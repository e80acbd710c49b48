#!/usr/bin/env python
"""The LIBERO pretraining recipe (scripts/LIBERO/DreamVLA/pretrain.sh: 24 layers, D 1024, S = 11, obs head, MLP action head,
--gripper_width, --atten_only_obs --mask_l_obs_ratio 0.5, --precision fp32, batch 10, accumulation 8 with the reference's
exchange every micro-step) on one GPU, as one JSON line:

  * time per micro-step and samples/s of three variants, timed with CUDA events in alternating rounds after warm-up:
      eager_host    eager TrainStep, the mask drawn with np.random on the host (the reference's sequence; one
                    device-to-host read and two uploads per forward),
      eager_device  eager TrainStep, the mask drawn on the device (DreamVLA.obs_drop_on_device),
      graphed       GraphedTrainStep (switches to the device draw itself; one replay per micro-step);
    the two eager variants share one model, the graphed variant has its own;
  * the draw alone (ops.ObsDropMask.draw: the drop kernel + the tile-flag kernel) over many launches.

  python tools/prof_pretrain.py [--batch 10] [--steps 16] [--warmup 8] [--rounds 3] [--draws 2000]

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

MODEL = dict(sequence_length=11, num_resampler_query=16, num_obs_token_per_image=9, obs_pred=True, atten_only_obs=True,
             attn_robot_proprio_state=True, atten_goal=4, atten_goal_state=True, mask_l_obs_ratio=0.5, action_pred_steps=3,
             transformer_layers=24, hidden_dim=1024, transformer_heads=16, phase="pretrain", gripper_width=True,
             use_dit_head=False, attn_implementation="sdpa")
STEP = dict(sequence_length=11, future_steps=3, action_pred_steps=3, atten_goal=4, use_dit_head=False, loss_action=True,
            loss_image=True, gradient_accumulation_steps=8, learning_rate=1e-4, weight_decay=1e-4, gripper_width=True,
            reduce_every_micro_step=True)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), (x.strip() for x in out.split(","))))
    except (OSError, subprocess.SubprocessError) as e:
        return {"name": torch.cuda.get_device_name(0), "nvidia_smi_error": repr(e)}


def train_step(dev):
    """pretrain.sh's model (dropout 0.1, the GPT-2 default it trains with) and an fp32-master TrainStep on it."""
    from bench import build_model
    from dreamvla_b200.utils.train_utils import StepConfig, TrainStep
    model = build_model({"model": MODEL}, dev, dropout=0.1)
    model.vision_encoder.requires_grad_(False)           # train.py: the ViT runs under no_grad
    master = {n: p.detach().float() for n, p in model.named_parameters() if p.requires_grad}
    return TrainStep(model, StepConfig(**STEP), master=master)


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def draw_time(dev, launches, rounds=5):
    """Per-draw ms of ops.ObsDropMask.draw at pretrain.sh's layout (K = 11, 57 slots, 18 observation tokens, count 9)."""
    from dreamvla_b200 import ops
    from dreamvla_b200.models.dreamvla_model import generate_attention_mask
    kw = dict(K=11, num_A=36, num_B=18 + 3, atten_goal=4, atten_goal_state=True, atten_only_obs=True,
              attn_robot_proprio_state=True, mask_l_obs_ratio=0.0, num_obs_token=18, action_pred_steps=3)
    m = ops.ObsDropMask(generate_attention_mask(**kw) == 0, dev, K=11, num_A=36, n_obs=18, n_act=3, count=9, seed=1)
    ctr = torch.zeros(1, dtype=torch.int64, device=dev)
    for _ in range(20):
        m.draw(ctr)
    torch.cuda.synchronize()
    per = max(1, launches // rounds)
    ts = [timed(lambda: m.draw(ctr), per) for _ in range(rounds)]
    return {"ms": round(statistics.median(ts), 5), "ms_min": round(min(ts), 5), "ms_max": round(max(ts), 5),
            "timed_draws": per * rounds, "L": m.Lq}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=10)
    ap.add_argument("--steps", type=int, default=16, help="timed micro-steps per variant and round")
    ap.add_argument("--warmup", type=int, default=8, help="untimed micro-steps per variant before each timed window")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--draws", type=int, default=2000, help="timed launches of the draw alone")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_pretrain.py needs a GPU")
    from dreamvla_b200.utils.train_utils import GraphedTrainStep, synthetic_batch
    dev = torch.device("cuda:0")
    info_before = gpu_info()
    eager = train_step(dev)
    graphed = GraphedTrainStep(train_step(dev), synthetic_batch(eager.cfg, args.batch, dev, seed=99), warmup=3)
    batch = synthetic_batch(eager.cfg, args.batch, dev, seed=99)

    def use_device_draw(on):
        eager.model.obs_drop_on_device = on

    variants = {"eager_host": (lambda: use_device_draw(False), lambda: eager(batch)),
                "eager_device": (lambda: use_device_draw(True), lambda: eager(batch)),
                "graphed": (lambda: None, lambda: graphed(batch))}
    times = {k: [] for k in variants}
    for r in range(args.rounds):
        for name, (setup, step) in variants.items():
            setup()
            for _ in range(args.warmup):
                step()
            torch.cuda.synchronize()
            times[name].append(timed(step, args.steps))
            print(f"[prof_pretrain] round {r} {name}: {times[name][-1]:.2f} ms/micro-step", file=sys.stderr, flush=True)
    loss_ok = bool(torch.isfinite(graphed.loss).all())
    kern = draw_time(dev, args.draws)
    info_after = gpu_info()
    res = {}
    for name, ts in times.items():
        ms = statistics.median(ts)
        res[name] = {"ms_per_micro_step": round(ms, 2), "ms_min": round(min(ts), 2), "ms_max": round(max(ts), 2),
                     "samples_per_s": round(args.batch / ms * 1e3, 2)}
    line = {"tool": "prof_pretrain", "gpu": info_before.get("name"), "power_limit": info_before.get("power.limit"),
            "sm_clock_mhz_before": info_before.get("clocks.sm"), "sm_clock_mhz_after": info_after.get("clocks.sm"),
            "sm_clock_max_mhz": info_before.get("clocks.max.sm"), "batch": args.batch,
            "accumulation": STEP["gradient_accumulation_steps"], "timed_micro_steps_per_round": args.steps,
            "rounds": args.rounds, "variants": res, "draw": kern, "graphed_loss_finite": loss_ok}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
