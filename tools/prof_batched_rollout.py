#!/usr/bin/env python
"""Throughput of batched rollouts on one GPU: `num_envs` simulated envs served per batched step (BatchedModelWrapper), as one
JSON line, for two models

  * eval.sh:  CALVIN eval.sh's model (bench.py's LATENCY_MODEL: obs + depth + SAM heads, DiT-B, S = 10), CALVIN wrapper;
  * libero:   the LIBERO scripts' model (world heads off, --gripper_width, DiT-B, S = 7), LIBERO wrapper;

at N in {1, 2, 4, 8}:

  * step: p50 / p99 per batched step and actions/s (N / p50), incremental (`rollout_actions`) and full window (a batch-N
    `mode='test'` forward), CUDA graphs on, envs starting staggered so that a batch mixes window fill levels
    (`rollout_bench.run_batched`, host clock around each step with a device synchronise on both sides).  The actions of
    N = 1 come from the fused sampler kernel, those of N >= 2 from the module sampler.

Rounds alternate the models and, within a round, the order of N; each round builds its model afresh.  Medians over rounds are
reported with their range.  The GPU's name, power limit and SM clocks are read in the same run.

  python tools/prof_batched_rollout.py [--rounds 2] [--steps 40] [--skip 10]
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

NS = (1, 2, 4, 8)
MODES = ("incremental", "full_window")


def model_cfg(name):
    from bench import LATENCY_MODEL
    if name == "eval.sh":
        return dict(LATENCY_MODEL)
    return dict(LATENCY_MODEL, sequence_length=7, obs_pred=False, depth_pred=False, sam_feat_pred=False, gripper_width=True)


def build(name, dev):
    from dreamvla_b200.models import DreamVLA
    torch.manual_seed(0)
    model = DreamVLA(finetune_type="calvin", clip_device="cpu", vit_checkpoint_path=None, **model_cfg(name)).bfloat16().to(dev)
    model._init_model_type()
    return model.eval()


def wrapper(name, model, n, mode, dev):
    S = model.sequence_length
    if name == "eval.sh":
        from dreamvla_b200.utils.eval_utils_calvin import BatchedModelWrapper
        return BatchedModelWrapper(model, n, history_len=S, device=dev, incremental=mode == "incremental")
    from dreamvla_b200.utils.eval_utils_libero import BatchedModelWrapper
    return BatchedModelWrapper(model, n, history_len=S, gripper_width=True, device=dev, incremental=mode == "incremental")


def round_for(name, dev, r, args):
    from dreamvla_b200.utils import rollout_bench
    model = build(name, dev)
    kind = "calvin" if name == "eval.sh" else "libero"
    out = {}
    for n in (NS if r % 2 == 0 else NS[::-1]):
        for mode in (MODES if r % 2 == 0 else MODES[::-1]):
            w = wrapper(name, model, n, mode, dev)
            lat = rollout_bench.run_batched(w, args.steps, kind, seed=1, episode_len=2 * model.sequence_length + 3)
            out[f"{mode}_n{n}"] = rollout_bench.batched_report(lat, args.skip, n, mode)
            del w
            torch.cuda.empty_cache()
    del model
    torch.cuda.empty_cache()
    return out


def main():
    from prof_pretrain import gpu_info
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=40, help="batched steps per model, N, mode and round")
    ap.add_argument("--skip", type=int, default=10, help="leading steps left out of the percentiles (graph capture)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_batched_rollout.py needs a GPU")
    dev = torch.device("cuda:0")
    info_before = gpu_info()
    names = ("eval.sh", "libero")
    rounds = {m: [] for m in names}
    for r in range(args.rounds):
        for m in (names if r % 2 == 0 else names[::-1]):
            rounds[m].append(round_for(m, dev, r, args))
            x = rounds[m][-1]
            print(f"[prof_batched_rollout] round {r} {m}: " + ", ".join(
                f"N={n} inc p50 {x[f'incremental_n{n}']['p50']:.2f} ms / full {x[f'full_window_n{n}']['p50']:.2f} ms"
                for n in NS), file=sys.stderr, flush=True)
    info_after = gpu_info()

    def med(vals, nd=3):
        vals = [v for v in vals if v is not None]
        if not vals:
            return None, None
        return round(statistics.median(vals), nd), [round(min(vals), nd), round(max(vals), nd)]
    res = {}
    for m in names:
        res[m] = {}
        for n in NS:
            for mode in MODES:
                for q in ("p50", "p99", "actions_per_s"):
                    res[m][f"{mode}_n{n}_{q}"], res[m][f"{mode}_n{n}_{q}_range"] = med([x[f"{mode}_n{n}"][q] for x in rounds[m]])
    print(json.dumps({"tool": "prof_batched_rollout", "gpu": info_before.get("name"), "power_limit": info_before.get("power.limit"),
                      "sm_clock_mhz_before": info_before.get("clocks.sm"), "sm_clock_mhz_after": info_after.get("clocks.sm"),
                      "sm_clock_max_mhz": info_before.get("clocks.max.sm"), "steps": args.steps, "skip": args.skip,
                      "rounds": args.rounds, "results": res}))


if __name__ == "__main__":
    main()
