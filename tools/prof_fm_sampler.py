#!/usr/bin/env python
"""Latency of flow-matching (`--use_fm`) action inference on one GPU, fused sampler (csrc/dit_sampler.cu, Euler integrator)
against the module path (FMDiffusion.ddim_sample_loop over the DiT modules), for the DiT-S, DiT-B and DiT-L action heads, as
one JSON line:

  * rollout: batch-1 incremental `ModelWrapper.step` p50 / p99 (bench.py's action-latency model, CALVIN eval.sh's, with
    use_fm=True; CUDA graphs on, prune=True), timed host-side around each call by `rollout_bench.run_calvin`;
  * sampler: `DreamVLA._ddim_actions` alone on one sequence, as tools/prof_sampler.py times it: the fused kernel called
    eagerly, the launch-bound module path replayed as a CUDA graph (the way the wrapper runs it); CUDA events over many calls.

Rounds alternate the sizes (DiT-S, DiT-B, DiT-L, DiT-S, ...) and, within a size, the order of the two variants; each round
builds its model afresh, so only one model is resident at a time.  The medians over rounds are reported with their range.

  python tools/prof_fm_sampler.py [--rounds 2] [--latency-steps 120] [--latency-skip 20] [--sampler-iters 50]

The GPU's name, power limit and SM clocks are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

DIT_TYPES = ("DiT-S", "DiT-B", "DiT-L")
VARIANTS = ("fused", "module")


def build(dit_type, dev):
    from bench import LATENCY_MODEL
    from dreamvla_b200.models import DreamVLA
    torch.manual_seed(0)
    model = DreamVLA(finetune_type="calvin", clip_device="cpu", vit_checkpoint_path=None,
                     **dict(LATENCY_MODEL, dit_type=dit_type, use_fm=True)).bfloat16().to(dev)
    model._init_model_type()
    return model.eval()


def sampler_ms(model, fused, dev, iters):
    """ms per `_ddim_actions` call on one sequence: fused eagerly (one launch), module as a CUDA-graph replay."""
    from prof_pretrain import timed
    g = torch.Generator().manual_seed(1)
    feat = (torch.randn(1, 3, 1024, generator=g) * 0.7).to(dev, torch.bfloat16)
    start = torch.randn(1, 3, 7, generator=g).to(dev)
    model.FUSED_SAMPLER = fused
    with torch.no_grad():
        for _ in range(3):
            model._ddim_actions(feat, start, dev)
        torch.cuda.synchronize()
        run = lambda: model._ddim_actions(feat, start, dev)       # noqa: E731
        if not fused:
            graph = torch.cuda.CUDAGraph()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                model._ddim_actions(feat, start, dev)
            torch.cuda.current_stream().wait_stream(side)
            with torch.cuda.graph(graph):
                model._ddim_actions(feat, start, dev)
            run = graph.replay
        run()
        torch.cuda.synchronize()
        return timed(run, iters)


def round_for(dit_type, dev, r, args):
    from bench import LATENCY_MODEL
    from dreamvla_b200.utils import rollout_bench
    from dreamvla_b200.utils.eval_utils_calvin import ModelWrapper
    model = build(dit_type, dev)
    out = {}
    for v in (VARIANTS if r % 2 == 0 else VARIANTS[::-1]):
        model.FUSED_SAMPLER = v == "fused"
        w = ModelWrapper(model, history_len=LATENCY_MODEL["sequence_length"], action_pred_steps=3, device=dev, incremental=True,
                         prune=True)
        lat = rollout_bench.run_calvin(w, args.latency_steps, seed=1)
        out[f"step_incremental_{v}"] = rollout_bench.percentile_report(lat, skip=args.latency_skip)
        del w
        out[f"sampler_{v}_ms"] = sampler_ms(model, v == "fused", dev, args.sampler_iters)
    del model
    torch.cuda.empty_cache()
    return out


def main():
    from prof_pretrain import gpu_info
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--latency-steps", type=int, default=120, help="ModelWrapper.step calls per variant, size and round")
    ap.add_argument("--latency-skip", type=int, default=20, help="leading calls left out of the percentiles")
    ap.add_argument("--sampler-iters", type=int, default=50, help="timed sampler calls per variant, size and round")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_fm_sampler.py needs a GPU")
    dev = torch.device("cuda:0")
    info_before = gpu_info()
    rounds = {t: [] for t in DIT_TYPES}
    for r in range(args.rounds):
        for t in DIT_TYPES:
            rounds[t].append(round_for(t, dev, r, args))
            x = rounds[t][-1]
            print(f"[prof_fm_sampler] round {r} {t}: " + ", ".join(
                f"{v}: step p50 {x[f'step_incremental_{v}']['p50']:.2f} ms, sampler {x[f'sampler_{v}_ms']:.3f} ms" for v in VARIANTS),
                file=sys.stderr, flush=True)
    info_after = gpu_info()

    def med(vals, nd=3):
        return round(statistics.median(vals), nd), [round(min(vals), nd), round(max(vals), nd)]
    res = {}
    for t in DIT_TYPES:
        res[t] = {}
        for v in VARIANTS:
            for q in ("p50", "p99"):
                res[t][f"step_incremental_{v}_{q}_ms"], res[t][f"step_incremental_{v}_{q}_range"] = med(
                    [x[f"step_incremental_{v}"][q] for x in rounds[t]])
            res[t][f"sampler_{v}_ms"], res[t][f"sampler_{v}_range"] = med([x[f"sampler_{v}_ms"] for x in rounds[t]])
        res[t]["fused_p50_below_module_p50"] = res[t]["step_incremental_fused_p50_ms"] < res[t]["step_incremental_module_p50_ms"]
    line = {"tool": "prof_fm_sampler", "gpu": info_before.get("name"), "power_limit": info_before.get("power.limit"),
            "sm_clock_mhz_before": info_before.get("clocks.sm"), "sm_clock_mhz_after": info_after.get("clocks.sm"),
            "sm_clock_max_mhz": info_before.get("clocks.max.sm"), "latency_steps_per_variant": args.latency_steps,
            "latency_skip": args.latency_skip, "sampler_iters": args.sampler_iters, "rounds": args.rounds, "results": res}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
