#!/usr/bin/env python
"""Cost of the action-head size (`--dit_type` DiT-S / DiT-B / DiT-L) on one GPU, as one JSON line:

  * train: the graphed C3 train step (bench.py's `libero` config: LIBERO, world heads off, S = 7, 24 layers) at batch 16,
    samples/s timed with CUDA events;
  * rollout: batch-1 `ModelWrapper.step` p50 / p99 (bench.py's action-latency workload, CALVIN eval.sh's model), full-window
    and incremental, once with the fused DDIM sampler (csrc/dit_sampler.cu) and once with the module path.

Rounds alternate the three sizes (DiT-S, DiT-B, DiT-L, DiT-S, ...); each round builds its model afresh, so only one model is
resident at a time.  The medians over rounds are reported with their range.

  python tools/prof_dit_type.py [--rounds 2] [--steps 10] [--warmup 3] [--latency-steps 120]

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


def train_round(dit_type, dev, batch, steps, warmup):
    from bench import CONFIGS, build_model
    from prof_pretrain import timed
    from dreamvla_b200.utils.train_utils import GraphedTrainStep, StepConfig, TrainStep, synthetic_batch
    cfg = CONFIGS["libero"]
    scfg = StepConfig(**cfg["step"])
    model = build_model({"model": dict(cfg["model"], dit_type=dit_type)}, dev, dropout=0.1)
    data = synthetic_batch(scfg, batch, dev, seed=99, heads=dict(cfg["heads"], flow_mask=scfg.flow_as_mask))
    step = GraphedTrainStep(TrainStep(model, scfg), data, warmup=3)
    for _ in range(warmup):
        step(step.static)
    torch.cuda.synchronize()
    ms = timed(lambda: step(step.static), steps)
    finite = bool(torch.isfinite(step.loss).all())
    del step, model
    torch.cuda.empty_cache()
    return ms, finite


def latency_round(dit_type, dev, steps, skip):
    from bench import LATENCY_MODEL
    from dreamvla_b200.models import DreamVLA
    from dreamvla_b200.utils import rollout_bench
    from dreamvla_b200.utils.eval_utils_calvin import ModelWrapper
    torch.manual_seed(0)
    model = DreamVLA(finetune_type="calvin", clip_device="cpu", vit_checkpoint_path=None,
                     **dict(LATENCY_MODEL, dit_type=dit_type)).bfloat16().to(dev)
    model._init_model_type()
    model.eval()
    out = {}
    for fused in (True, False):
        model.FUSED_SAMPLER = fused
        for name, kw in (("full_window", dict(incremental=False)), ("incremental", dict(incremental=True, prune=True))):
            w = ModelWrapper(model, history_len=LATENCY_MODEL["sequence_length"], action_pred_steps=3, device=dev, **kw)
            lat = rollout_bench.run_calvin(w, steps, seed=1)
            out[f"{name}_{'fused' if fused else 'module'}"] = rollout_bench.percentile_report(lat, skip=skip)
            del w
    del model
    torch.cuda.empty_cache()
    return out


def main():
    from prof_pretrain import gpu_info
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", type=int, default=10, help="timed graphed train steps per size and round")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--latency-steps", type=int, default=120, help="ModelWrapper.step calls per variant, size and round")
    ap.add_argument("--latency-skip", type=int, default=20, help="leading calls left out of the percentiles")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_dit_type.py needs a GPU")
    dev = torch.device("cuda:0")
    info_before = gpu_info()
    train_ms = {t: [] for t in DIT_TYPES}
    finite = {t: True for t in DIT_TYPES}
    lat = {t: [] for t in DIT_TYPES}
    for r in range(args.rounds):
        for t in DIT_TYPES:
            ms, ok = train_round(t, dev, args.batch, args.steps, args.warmup)
            train_ms[t].append(ms)
            finite[t] = finite[t] and ok
            print(f"[prof_dit_type] round {r} {t}: train {ms:.2f} ms/step", file=sys.stderr, flush=True)
        for t in DIT_TYPES:
            lat[t].append(latency_round(t, dev, args.latency_steps, args.latency_skip))
            print(f"[prof_dit_type] round {r} {t}: " + ", ".join(f"{k} p50 {v['p50']:.2f} ms" for k, v in lat[t][-1].items()),
                  file=sys.stderr, flush=True)
    info_after = gpu_info()
    res = {}
    for t in DIT_TYPES:
        ms = statistics.median(train_ms[t])
        res[t] = {"train_ms_per_step": round(ms, 2), "train_ms_range": [round(min(train_ms[t]), 2), round(max(train_ms[t]), 2)],
                  "train_samples_per_s": round(args.batch / ms * 1e3, 2), "train_loss_finite": finite[t]}
        for k in lat[t][0]:
            for q in ("p50", "p99"):
                v = [x[k][q] for x in lat[t]]
                res[t][f"step_{k}_{q}_ms"] = round(statistics.median(v), 3)
                res[t][f"step_{k}_{q}_range"] = [round(min(v), 3), round(max(v), 3)]
    line = {"tool": "prof_dit_type", "gpu": info_before.get("name"), "power_limit": info_before.get("power.limit"),
            "sm_clock_mhz_before": info_before.get("clocks.sm"), "sm_clock_mhz_after": info_after.get("clocks.sm"),
            "sm_clock_max_mhz": info_before.get("clocks.max.sm"), "train_batch": args.batch, "train_steps_per_round": args.steps,
            "latency_steps_per_variant": args.latency_steps, "latency_skip": args.latency_skip, "rounds": args.rounds,
            "results": res}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
