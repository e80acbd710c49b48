"""Cost of CLIP's image transform on the device (dvla_image_fn, `data_utils.preprocess_image`) and what it buys:

  python tools/prof_image_fn.py [--out results/prof_image_fn.json] [--skip-train] [--skip-rollout]

1. kernel time (CUDA events over >= 100 warm launches) of one training step's frames: C2 (B=8, 13-frame windows: 104 frames of
   200x200 + 104 of 84x84) and C3 (B=16, 10-frame windows: 320 frames of 128x128), bf16 out; achieved bandwidth from the bytes
   the shapes imply (uint8 frames read + output written) against the H100 SXM data-sheet 3.35 TB/s;
2. the C3 training loop at B=16 (CUDA-graph step, copy-stream prefetch from pinned host memory) fed fp32 preprocessed frames
   vs uint8 raw frames, alternated in one run;
3. CALVIN rollout latency (eval.sh model, batch 1) with raw 200x200 / 84x84 frames -- preprocessing included -- vs
   preprocessed tensors, full-window and incremental.
The card name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBS = 3.35


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q}


def kernel_times(dev, iters=200):
    from dreamvla_b200.utils.data_utils import preprocess_image
    cases = {"C2 step (104 x 200^2 + 104 x 84^2)": [(104, 200, 200), (104, 84, 84)], "C3 step (320 x 128^2)": [(320, 128, 128)]}
    out = {}
    g = torch.Generator().manual_seed(0)
    for name, shapes in cases.items():
        for dt in (torch.bfloat16, torch.float32):
            frames = [torch.randint(0, 256, (n, h, w, 3), generator=g, dtype=torch.uint8).to(dev) for n, h, w in shapes]
            run = lambda: [preprocess_image(f, dt) for f in frames]        # noqa: E731
            for _ in range(20):
                run()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                run()
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / iters
            nbytes = sum(n * h * w * 3 + n * 3 * 224 * 224 * (2 if dt == torch.bfloat16 else 4) for n, h, w in shapes)
            out[f"{name} -> {str(dt).split('.')[-1]}"] = {
                "us_per_step": round(us, 2), "launches_per_step": len(shapes), "bytes": nbytes,
                "GB_per_s": round(nbytes / us / 1e3, 1), "frac_of_3.35TBps": round(nbytes / us / 1e6 / HBM_TBS, 3)}
    return out


def train_loop(dev, rounds=3, steps=12):
    import bench
    from dreamvla_b200.utils.data_utils import prepare_batch
    from dreamvla_b200.utils.train_utils import GraphedTrainStep, StepConfig, TrainStep, prefetch_to_device, synthetic_batch
    cfg = bench.CONFIGS["libero"]
    scfg = StepConfig(**cfg["step"])
    B, W = 16, scfg.sequence_length + scfg.future_steps
    model = bench.build_model(cfg, dev, 0.1)
    base = synthetic_batch(scfg, B, "cpu", seed=3, dtype=torch.float32)
    g = torch.Generator().manual_seed(4)
    raw = {"images_primary": torch.randint(0, 256, (B, W, 128, 128, 3), generator=g, dtype=torch.uint8),
           "images_wrist": torch.randint(0, 256, (B, W, 128, 128, 3), generator=g, dtype=torch.uint8)}
    host_raw = {k: v.pin_memory() for k, v in dict(base, **raw).items()}
    pre = prepare_batch({k: v.to(dev) for k, v in raw.items()}, dtype=torch.float32)
    host_f32 = {k: v.pin_memory() for k, v in dict(base, **{k: v.cpu() for k, v in pre.items()}).items()}
    step = GraphedTrainStep(TrainStep(model, scfg), prepare_batch({k: v.to(dev) for k, v in host_raw.items()}), warmup=3)

    def run(host, n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for batch in prefetch_to_device([host] * n, dev):
            loss = step(prepare_batch(batch))
        torch.cuda.synchronize()
        return B * n / (time.perf_counter() - t0), float(loss)

    run(host_f32, 3)
    run(host_raw, 3)
    res = {"fp32_preprocessed": [], "uint8_raw": []}
    for _ in range(rounds):
        res["fp32_preprocessed"].append(round(run(host_f32, steps)[0], 2))
        res["uint8_raw"].append(round(run(host_raw, steps)[0], 2))
    h2d = {k: sum(v.numel() * v.element_size() for kk, v in h.items() if kk.startswith("images"))
           for k, h in (("fp32_preprocessed", host_f32), ("uint8_raw", host_raw))}
    del step, model
    torch.cuda.empty_cache()
    return {"workload": "C3 LIBERO train step B=16, CUDA graph, copy-stream prefetch from pinned host", "unit": "samples/s",
            "steps_per_round": steps, "rounds": res, "image_bytes_per_step_h2d": h2d}


def rollout(dev, steps=300, skip=25):
    import bench
    from dreamvla_b200.models import DreamVLA
    from dreamvla_b200.utils import rollout_bench
    from dreamvla_b200.utils.eval_utils_calvin import ModelWrapper
    torch.manual_seed(0)
    model = DreamVLA(finetune_type="calvin", clip_device="cpu", vit_checkpoint_path=None, **bench.LATENCY_MODEL).bfloat16().to(dev)
    model._init_model_type()
    model.eval()
    text = rollout_bench.synthetic_text(1)

    def run_raw(w):
        g = torch.Generator().manual_seed(1)
        lat = []
        for i in range(steps):
            if i % 360 == 0:
                w.reset()
            img = torch.randint(0, 256, (200, 200, 3), generator=g, dtype=torch.uint8).numpy()
            grip = torch.randint(0, 256, (84, 84, 3), generator=g, dtype=torch.uint8).numpy()
            obs = torch.randn(15, generator=g)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            w.step(img, grip, obs, text)
            torch.cuda.synchronize()
            lat.append((time.perf_counter() - t0) * 1e3)
        return lat

    out = {"workload": "CALVIN action inference (eval.sh model), batch 1", "unit": "ms"}
    for name, kw in (("full_window", dict(incremental=False)), ("incremental", dict(incremental=True, prune=True))):
        w = ModelWrapper(model, history_len=10, action_pred_steps=3, device=dev, **kw)
        out[name] = {"preprocessed_tensors": rollout_bench.percentile_report(rollout_bench.run_calvin(w, steps, seed=1), skip),
                     "raw_uint8_frames": rollout_bench.percentile_report(run_raw(w), skip)}
        del w
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip-train", action="store_true")
    ap.add_argument("--skip-rollout", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_image_fn.py measures on a GPU; none is visible")
    dev = torch.device("cuda:0")
    res = {"card": card(), "kernel": kernel_times(dev)}
    print(json.dumps(res, indent=1), flush=True)
    if not a.skip_train:
        res["train_loop"] = train_loop(dev)
        print(json.dumps(res["train_loop"], indent=1), flush=True)
    if not a.skip_rollout:
        res["rollout"] = rollout(dev)
        print(json.dumps(res["rollout"], indent=1), flush=True)
    res["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
