"""Checks that two builds of the library compute bit-identical attention gradients.

  python tools/attn_bwd_identity.py --ref PARENT.so [--lib NEW.so] [--json OUT]

Runs the forward and backward of every case below once per library, each library in a subprocess of its own (the way
`tools/prof_attention.py --lib` loads one), and compares o, lse, dq, dk and dv with torch.equal.  `--lib` defaults to
dreamvla_b200/lib/libdvla_sm90.so.  Cases: the backward cases of tests/test_attn_wgmma_gpu.py, the production shapes of the
CALVIN train step (backbone 8 x 16 x 1290 under its block mask with attention dropout 0.1 and 0, decoder 160 x 16 x 265),
one short-query case on the mma.sync backward (which shares the dQ-form element-wise helper), and the edges of the
backward's persistent schedule: more work units than CTAs at an odd tile count, a single (b, h), and
an SM budget below the device's (dvla_set_sm_budget).  Exits non-zero if any tensor differs."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

SCALE = 0.125
SEED = 0x5EED0FA77E57
# (id, B, H, Lq, Lk, mask, dropout p, SM budget or 0): mask None, "backbone" or "random" as in test_attn_wgmma_gpu.py
CASES = [
    ("backbone_8x16x1290_p0.1", 8, 16, 1290, 1290, "backbone", 0.1, 0),
    ("backbone_8x16x1290_p0", 8, 16, 1290, 1290, "backbone", 0.0, 0),
    ("backbone_2x16x1290_p0", 2, 16, 1290, 1290, "backbone", 0.0, 0),
    ("decoder_160x16x265", 160, 16, 265, 265, None, 0.0, 0),
    ("decoder_160x16x265_p0.1", 160, 16, 265, 265, None, 0.1, 0),
    ("lq96_p0.1", 2, 3, 96, 96, None, 0.1, 0),
    ("lq96_lk200_random_p0.1", 2, 2, 96, 200, "random", 0.1, 0),
    ("lq330_lk140_random_p0.1", 2, 2, 330, 140, "random", 0.1, 0),
    ("lq256_lk320_random_p0", 1, 3, 256, 320, "random", 0.0, 0),
    ("lq200_lk517_p0.3", 2, 2, 200, 517, None, 0.3, 0),
    ("mma_sync_lq80_lk200_random_p0.1", 2, 2, 80, 200, "random", 0.1, 0),
    ("odd_tiles_40x8x300_random_p0.1", 40, 8, 300, 300, "random", 0.1, 0),
    ("single_bh_1x1x1290_p0.1", 1, 1, 1290, 1290, "backbone", 0.1, 0),
    ("budget40_decoder_32x16x265_p0.1", 32, 16, 265, 265, None, 0.1, 40),
]


def _vis(mask, Lq, Lk, g):
    if mask == "backbone":
        from dreamvla_b200.models.dreamvla_model import generate_attention_mask
        add = generate_attention_mask(K=10, num_A=36, num_B=93, atten_goal=0, atten_goal_state=False, atten_only_obs=False,
                                      attn_robot_proprio_state=False, mask_l_obs_ratio=0.0, num_obs_token=90,
                                      action_pred_steps=3)
        return add == 0
    if mask == "random":
        m = torch.rand(Lq, Lk, generator=g) < 0.3
        m[:, 0] = True
        m[: Lq // 2, 64:128] = False
        m[Lq // 2:, 64:128] = True
        return m
    return None


def dump(lib_path, out):
    from dreamvla_b200 import _lib as L
    from dreamvla_b200 import ops
    L.LIB_PATH = os.path.abspath(lib_path)
    L.load()
    dev = torch.device("cuda:0")
    res = {}
    for name, B, H, Lq, Lk, mask, p, budget in CASES:
        g = torch.Generator().manual_seed(B * 7919 + Lq * 31 + Lk)
        vis = _vis(mask, Lq, Lk, g)
        am = ops.AttnMask(vis, dev) if vis is not None else None
        bits, flags = (am.bits, am.flags) if am is not None else (None, None)
        q, k, v = (torch.randn(B, n, H, 64, generator=g).to(dev, torch.bfloat16) for n in (Lq, Lk, Lk))
        d_o = torch.randn(B, Lq, H, 64, generator=g).to(dev, torch.bfloat16)
        prev = L.set_sm_budget(budget) if budget else None
        try:
            o, lse = L.attn_fwd(q, k, v, SCALE, bits, flags, dropout_p=p, dropout_seed=SEED)
            dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
            L.attn_bwd(q, k, v, o, d_o, lse, SCALE, dq, dk, dv, bits, flags, dropout_p=p, dropout_seed=SEED)
            torch.cuda.synchronize()
        finally:
            if budget:
                L.set_sm_budget(prev)
        res[name] = {n: t.cpu() for n, t in zip(("o", "lse", "dq", "dk", "dv"), (o, lse, dq, dk, dv))}
    torch.save(res, out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", required=True, help="the library to compare against (e.g. the parent commit's build)")
    ap.add_argument("--lib", default=os.path.join(ROOT, "dreamvla_b200", "lib", "libdvla_sm90.so"))
    ap.add_argument("--json", default=None)
    ap.add_argument("--dump", default=None, help=argparse.SUPPRESS)   # subprocess mode: run CASES on --lib into this file
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_bwd_identity.py runs the CUDA kernels and needs a GPU")
    if args.dump:
        dump(args.lib, args.dump)
        return
    with tempfile.TemporaryDirectory() as tmp:
        outs = []
        for i, lib in enumerate((args.ref, args.lib)):
            out = os.path.join(tmp, f"{i}.pt")
            subprocess.run([sys.executable, os.path.abspath(__file__), "--ref", args.ref, "--lib", lib, "--dump", out], check=True)
            outs.append(torch.load(out))
    ref, new = outs
    n_tensors, diffs = 0, []
    for name in ref:
        for t in ref[name]:
            n_tensors += 1
            if not torch.equal(ref[name][t], new[name][t]):
                d = (ref[name][t].float() - new[name][t].float()).abs()
                diffs.append({"case": name, "tensor": t, "elements": int((d != 0).sum()), "max_abs": float(d.max())})
    print(f"[identity] {args.lib} vs {args.ref}: {n_tensors} tensors over {len(ref)} cases, {len(diffs)} differ")
    for d in diffs:
        print("  " + json.dumps(d))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump({"ref": args.ref, "lib": args.lib, "tensors": n_tensors, "differ": diffs}, f, indent=1)
    sys.exit(1 if diffs else 0)


if __name__ == "__main__":
    main()
