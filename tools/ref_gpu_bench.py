"""Context number, NOT a bench arm: the reference's algorithm (oracle/, a functional PyTorch restatement) run on the GPU
the way the reference itself runs (PyTorch eager kernels + cuBLAS under torch.autocast(bf16), fp32 master weights,
torch.optim.AdamW, clip_grad_norm_) — BASELINE.md §3 "reference GPU build".  Prints one JSON line per batch size so that
a result can quote  ours / (stock PyTorch)  on the same GPU.  Test/measurement infrastructure: imports oracle/.

  python tools/ref_gpu_bench.py [--batch 2 8] [--sdpa] [--steps 5]
"""
import argparse
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from bench import CONFIGS  # noqa: E402
from oracle import dreamvla_oracle as O  # noqa: E402
from tests import synth  # noqa: E402
from tests.state_template import build_template  # noqa: E402


def _mha_sdpa(q, k, v, scale, mask=None):
    q, k, v = (t.permute(0, 2, 1, 3) for t in (q, k, v))
    if mask is not None:
        mask = mask.to(q.dtype)
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, scale=scale).permute(0, 2, 1, 3)
    return o.reshape(o.shape[0], o.shape[1], -1)


def run(batch, args):
    dev = torch.device("cuda:0")
    cfg = CONFIGS[args.config]
    mk = dict(cfg["model"], batch=batch, weight_seed=1, input_seed=2)
    sd = {k: v.to(dev) for k, v in synth.synth_state_dict(build_template(mk), 1).items()}
    frozen = ("vision_encoder.", "clip_model.", "attention_mask", "position_embedding")
    params = []
    for k, v in sd.items():
        if v.is_floating_point() and not any(f in k for f in frozen):
            v.requires_grad_(True)
            params.append(v)
    opt = torch.optim.AdamW(params, lr=1e-3, weight_decay=1e-4, fused=True)
    inp = {k: v.to(dev) for k, v in synth.synth_inputs(mk).items()}
    lab = {k: v.to(dev) for k, v in synth.synth_labels(mk).items()}
    S = mk["sequence_length"]
    n = 8 * batch * S
    noise = torch.randn(n, 3, 7, device=dev)
    tstep = torch.randint(0, 100, (n,), device=dev)
    drop = torch.rand(n, device=dev) < 0.1
    lcfg = dict(mk, future_steps=3, flow_as_mask=cfg["step"].get("flow_as_mask", False))

    def one():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            fwd = O.dreamvla_forward(sd, mk, inp["image_primary"], inp["image_wrist"], inp["state"], inp["text_token"],
                                     action_label=inp["action_label"], diffusion_noise=noise, diffusion_timestep=tstep,
                                     diffusion_drop_ids=drop)
            losses = O.train_losses(lcfg, fwd, lab)
        losses["loss"].backward()
        torch.nn.utils.clip_grad_norm_(params, 0.1)
        opt.step()
        return losses["loss"]

    for _ in range(args.warmup):
        one()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        loss = one()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    print(json.dumps({"impl": "oracle-on-gpu (torch eager + cuBLAS, autocast bf16)", "attention": "sdpa" if args.sdpa else "math",
                      "workload": cfg["name"], "batch": batch, "ms_per_step": round(ms, 2),
                      "samples_per_s": round(batch / ms * 1e3, 2), "loss": float(loss),
                      "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2**30, 2)}), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="calvin")
    ap.add_argument("--batch", type=int, nargs="+", default=[2, 8])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sdpa", action="store_true")
    args = ap.parse_args()
    if args.sdpa:
        O._mha = _mha_sdpa
    t0 = time.time()
    for b in args.batch:
        run(b, args)
        torch.cuda.empty_cache()
    print(f"# {time.time() - t0:.0f}s", flush=True)
