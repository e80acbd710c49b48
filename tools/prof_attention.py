"""Times the long-sequence attention kernels at the shapes the CALVIN train step (bench.py) runs them at.

  python tools/prof_attention.py [--lib PATH] [--iters N] [--step-table] [--json OUT]

Per case: the forward call and the backward call with CUDA events over `--iters` launches each, and the backward split
into its three kernels (delta, dK/dV, dQ) from a torch.profiler trace of `--iters` more calls.  Cases:
  backbone   8 x 16 heads x 1290, the GPT-2 block mask of the C2 step, attention dropout 0.1 and 0
  decoder    160 x 16 x 265, no mask, no dropout (world-knowledge decoders)
  vit        160 x 12 x 197, forward only (frozen ViT)
  per_seq    8 x 16 x 1290 forward under a two-mask stack selected per sequence (batched rollouts)
`--step-table` adds torch.profiler's kernel table of one eager C2 train step (bench.py's model at batch 8), so that
attention's share of the step is known.  `--lib` loads another build of the library (e.g. a parent commit's) instead of
dreamvla_b200/lib/libdvla_sm90.so.  The card's name, power limit and max SM clock are printed with the numbers."""
from __future__ import annotations

import argparse
import collections
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

SCALE = 0.125


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        out = ""
    return out or torch.cuda.get_device_name(0)


def backbone_mask():
    from dreamvla_b200.models.dreamvla_model import generate_attention_mask
    add = generate_attention_mask(K=10, num_A=36, num_B=93, atten_goal=0, atten_goal_state=False, atten_only_obs=False,
                                  attn_robot_proprio_state=False, mask_l_obs_ratio=0.0, num_obs_token=90, action_pred_steps=3)
    return add == 0


def time_events(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def kernel_split(fn, iters):
    """Device time per call of each kernel `fn` launches, from a torch.profiler trace of `iters` calls."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    tot = collections.defaultdict(float)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            tot[kernel_label(ev.name)] += ev.device_time / 1000.0
    return {k: v / iters for k, v in tot.items()}


def kernel_label(name):
    for key, label in (("attn_delta", "delta"), ("attn_bwd_wgmma_kernel<true>", "dkv"), ("attn_bwd_wgmma_kernel<(bool)1>", "dkv"),
                       ("attn_bwd_wgmma_kernel<false>", "dq"), ("attn_bwd_wgmma_kernel<(bool)0>", "dq"),
                       ("attn_fwd_wgmma", "fwd")):
        if key in name:
            return label
    return name[:60]


def run_cases(L, iters):
    from dreamvla_b200 import ops
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    res = {}
    vis = backbone_mask()
    am = ops.AttnMask(vis, dev)
    cases = [("backbone_p0.1", 8, 16, 1290, am, 0.1, True), ("backbone_p0", 8, 16, 1290, am, 0.0, True),
             ("decoder", 160, 16, 265, None, 0.0, True), ("vit", 160, 12, 197, None, 0.0, False)]
    for name, B, H, Lx, mask, p, bwd in cases:
        qkv = torch.randn(B, Lx, 3, H, 64, device=dev, dtype=torch.bfloat16, generator=g)
        q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
        bits, flags = (mask.bits, mask.flags) if mask is not None else (None, None)
        o, lse = L.attn_fwd(q, k, v, SCALE, bits, flags, dropout_p=p, dropout_seed=5)
        r = {"fwd_ms": time_events(lambda: L.attn_fwd(q, k, v, SCALE, bits, flags, dropout_p=p, dropout_seed=5), iters)}
        if bwd:
            d_o = torch.randn(o.shape, device=dev, dtype=torch.bfloat16, generator=g)
            dqkv = torch.empty_like(qkv)

            def call_bwd():
                L.attn_bwd(q, k, v, o, d_o, lse, SCALE, dqkv[:, :, 0], dqkv[:, :, 1], dqkv[:, :, 2], bits, flags,
                           dropout_p=p, dropout_seed=5)
            r["bwd_ms"] = time_events(call_bwd, iters)
            r["bwd_kernels_ms"] = kernel_split(call_bwd, iters)
        res[name] = r
        print(f"[attn] {name:14s} B{B} H{H} L{Lx} p={p}: " + json.dumps(r), flush=True)
    # per-sequence masks: the backbone mask and the same mask with the last step's observation keys hidden
    vis2 = vis.clone()
    vis2[:, -129:-39] = False
    vis2[torch.arange(vis.shape[0]), torch.arange(vis.shape[0])] = True
    stack = ops.AttnMaskStack(torch.stack([vis, vis2]), dev)
    idx = (torch.arange(8, device=dev) % 2).to(torch.int32)
    qkv = torch.randn(8, 1290, 3, 16, 64, device=dev, dtype=torch.bfloat16, generator=g)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    r = {"fwd_ms": time_events(lambda: L.attn_fwd(q, k, v, SCALE, stack.bits, stack.flags, mask_index=idx), iters)}
    res["per_seq"] = r
    print(f"[attn] per_seq        B8 H16 L1290 p=0.0: " + json.dumps(r), flush=True)
    return res


def step_table(rows=30):
    """torch.profiler kernel table of one eager C2 train step at batch 8 (bench.py's model, batch and step)."""
    import bench
    from torch.profiler import ProfilerActivity, profile
    from dreamvla_b200.utils.train_utils import StepConfig, TrainStep, synthetic_batch
    cfg = bench.CONFIGS["calvin"]
    dev = torch.device("cuda", 0)
    scfg = StepConfig(**cfg["step"])
    model = bench.build_model(cfg, dev, 0.1)
    step = TrainStep(model, scfg)
    batch = synthetic_batch(scfg, 8, dev, seed=1234, heads=dict(cfg["heads"], flow_mask=scfg.flow_as_mask))
    for _ in range(2):
        step(batch)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(batch)
        torch.cuda.synchronize()
    tot, cnt = collections.defaultdict(float), collections.Counter()
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            tot[ev.name] += ev.device_time / 1000.0
            cnt[ev.name] += 1
    total = sum(tot.values())
    attn = sum(v for k, v in tot.items() if "attn" in k)
    print(f"[step] eager C2 step, batch 8: kernel time {total:.2f} ms, attention kernels {attn:.2f} ms "
          f"({100 * attn / max(total, 1e-9):.1f} %)")
    for name, ms in sorted(tot.items(), key=lambda kv: -kv[1])[:rows]:
        print(f"  {ms:8.3f} ms {cnt[name]:5d}x  {name[:110]}")
    return {"kernel_ms": total, "attn_ms": attn,
            "attn_kernels_ms": {k[:110]: v for k, v in tot.items() if "attn" in k}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="library to load instead of dreamvla_b200/lib/libdvla_sm90.so")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--step-table", action="store_true")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_attention.py times CUDA kernels and needs a GPU")
    from dreamvla_b200 import _lib as L
    if args.lib:
        L.LIB_PATH = os.path.abspath(args.lib)
    L.load()
    out = {"card": card(), "lib": L.LIB_PATH}
    print(f"[card] {out['card']}  lib {L.LIB_PATH}", flush=True)
    out["cases"] = run_cases(L, args.iters)
    if args.step_table:
        out["step"] = step_table()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
