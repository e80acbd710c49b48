#!/usr/bin/env python
"""What fp32 master weights (`--precision fp32`) cost on one GPU, as one JSON line:

  * the optimiser kernels alone: dvla_adamw (bf16 parameters, 24 B per parameter) and dvla_adamw_master (fp32 masters + bf16
    working copy, 30 B per parameter) on flat buffers of the C2 trained-parameter count, alternating in one process, timed
    with CUDA events; achieved GB/s from those byte counts against the 3.35 TB/s HBM3 figure of NVIDIA's H100 SXM data sheet
    (a data-sheet number, not a measured peak);
  * the C2 train step (bench.py's CALVIN workload, CUDA-graph replay, device-resident synthetic batch) in bf16 mode and in fp32
    mode, each built, timed and freed in turn -- bf16, fp32, bf16, fp32 -- since two C2 replicas need not fit together.

  python tools/prof_master_weights.py [--batch 8] [--steps 20] [--kernel-launches 50]

The GPU's name, power limit and SM clocks are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

HBM_DATASHEET_TBPS = 3.35
BYTES_PER_PARAM = {"adamw": 24, "adamw_master": 30}


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), (x.strip() for x in out.split(","))))
    except (OSError, subprocess.SubprocessError) as e:
        return {"name": torch.cuda.get_device_name(0), "nvidia_smi_error": repr(e)}


def train_step_rate(mode, batch_size, steps, warmup, dev):
    """samples/s of the graphed C2 train step; everything it allocated is freed before it returns."""
    from bench import CONFIGS, build_model
    from dreamvla_b200.utils.train_utils import GraphedTrainStep, StepConfig, TrainStep, synthetic_batch
    cfg = CONFIGS["calvin"]
    scfg = StepConfig(**cfg["step"])
    model = build_model(cfg, dev, dropout=0.1)
    master = None
    if mode == "fp32":        # the bf16-initialised weights as fp32 masters: the values do not change the work
        master = {n: p.detach().float() for n, p in model.named_parameters() if p.requires_grad}
    eager = TrainStep(model, scfg, master=master)
    del master
    n_flat = eager.flat.n
    batch = synthetic_batch(scfg, batch_size, dev, seed=99, heads=dict(cfg["heads"], flow_mask=scfg.flow_as_mask))
    step = GraphedTrainStep(eager, batch, warmup=3)
    for _ in range(warmup):
        step(step.static)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step(step.static)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    out = {"mode": mode, "ms_per_step": round(ms, 3), "samples_per_s": round(batch_size / ms * 1e3, 3),
           "final_loss": round(float(loss), 5)}
    del step, eager, model, batch, loss
    torch.cuda.empty_cache()
    return out, n_flat


def optimizer_kernels(n, launches, dev, rounds=5):
    """Per-launch ms of dvla_adamw and dvla_adamw_master on n-element flat buffers, alternating in `rounds` rounds."""
    from dreamvla_b200 import _lib as L
    n = (n + 7) // 8 * 8
    g = torch.Generator(device=dev).manual_seed(0)
    P32 = torch.randn(n, device=dev, generator=g) * 0.02
    P = P32.to(torch.bfloat16)
    G = (torch.randn(n, device=dev, generator=g) * 1e-4).to(torch.bfloat16)
    m = torch.zeros(n, device=dev)
    v = torch.zeros(n, device=dev)
    ss = torch.ones(1, device=dev)
    lr = torch.full((1,), 1e-5, device=dev)
    st = torch.ones(1, device=dev)
    kw = dict(sumsq_t=ss, lr_t=lr, step_t=st, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=1e-4, max_norm=0.1,
              zero_grad=True)
    calls = {"adamw": lambda: L.adamw(P, G, m, v, **kw), "adamw_master": lambda: L.adamw_master(P32, P, G, m, v, **kw)}
    per = max(1, launches // rounds)
    for fn in calls.values():                 # warm-up: module load, first-touch of the buffers
        for _ in range(5):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in calls}
    for _ in range(rounds):
        for name, fn in calls.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(per):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / per)
    out = {}
    for name, ts in times.items():
        ms = statistics.median(ts)
        gbs = BYTES_PER_PARAM[name] * n / (ms * 1e-3) / 1e9
        out[name] = {"ms": round(ms, 4), "ms_min": round(min(ts), 4), "ms_max": round(max(ts), 4),
                     "timed_launches": per * rounds, "bytes_per_param": BYTES_PER_PARAM[name], "GB_per_s": round(gbs, 1),
                     "frac_of_datasheet_hbm": round(gbs / (HBM_DATASHEET_TBPS * 1e3), 3)}
    out["master_minus_bf16_ms"] = round(out["adamw_master"]["ms"] - out["adamw"]["ms"], 4)
    del P32, P, G, m, v
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--kernel-launches", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_master_weights.py needs a GPU")
    dev = torch.device("cuda:0")
    info_before = gpu_info()
    runs, n_flat = [], None
    for mode in ("bf16", "fp32", "bf16", "fp32"):
        r, n_flat = train_step_rate(mode, args.batch, args.steps, args.warmup, dev)
        runs.append(r)
        print(f"[prof_master_weights] {r}", file=sys.stderr, flush=True)
    kern = optimizer_kernels(n_flat, args.kernel_launches, dev)
    info_after = gpu_info()
    mean = {md: statistics.mean(r["samples_per_s"] for r in runs if r["mode"] == md) for md in ("bf16", "fp32")}
    line = {"tool": "prof_master_weights", "gpu": info_before.get("name"), "power_limit": info_before.get("power.limit"),
            "sm_clock_mhz_before": info_before.get("clocks.sm"), "sm_clock_mhz_after": info_after.get("clocks.sm"),
            "sm_clock_max_mhz": info_before.get("clocks.max.sm"), "flat_params": n_flat,
            "hbm_reference": f"{HBM_DATASHEET_TBPS} TB/s, NVIDIA H100 SXM data sheet (not measured)",
            "optimizer_kernels": kern,
            "train_step": {"workload": "C2 CALVIN train step, CUDA-graph replay, per-GPU batch %d" % args.batch,
                           "steps_per_run": args.steps, "runs": runs,
                           "bf16_samples_per_s": round(mean["bf16"], 3), "fp32_samples_per_s": round(mean["fp32"], 3),
                           "fp32_minus_bf16_samples_per_s": round(mean["fp32"] - mean["bf16"], 3),
                           "fp32_over_bf16": round(mean["fp32"] / mean["bf16"], 4)}}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
