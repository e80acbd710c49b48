#!/usr/bin/env python
"""Entry point mirroring reference eval_calvin.py:23-132 for the action-inference path.

The CALVIN simulator (PyBullet) is out of scope; `--synthetic_rollout_steps N` drives `ModelWrapper.step` with synthetic
observations and reports p50 / p99 per-action latency (the latency metric of BASELINE.json).  A real env can call
`dreamvla_b200.utils.eval_utils_calvin.ModelWrapper.step` exactly where the reference calls `model.step` (:264).
`--incremental_rollout` switches the wrapper to rollout-level incremental inference (per-frame token cache, SURVEY §8 f-1).
`--num_envs N` (N > 1) serves N envs per batched step (`BatchedModelWrapper`); with `--synthetic_rollout_steps` the N
synthetic envs start their episodes staggered and the report is per batched step, with actions/s.
Inference runs in bf16 whatever `--precision` says: the fp32 checkpoints of a `--precision fp32` run (and the reference's)
load by rounding each value to bf16.
"""
from __future__ import annotations

import json

import torch

from dreamvla_b200.models import DreamVLA
from dreamvla_b200.utils import rollout_bench
from dreamvla_b200.utils.arguments_utils import get_parser, model_kwargs
from dreamvla_b200.utils.eval_utils_calvin import BatchedModelWrapper, ModelWrapper


def load_model(args, dev):
    model = DreamVLA(finetune_type=args.finetune_type, clip_device="cpu", vit_checkpoint_path=args.vit_checkpoint_path,
                     **model_kwargs(args)).bfloat16().to(dev)
    model._init_model_type()
    if args.resume_from_checkpoint:
        ck = torch.load(args.resume_from_checkpoint, map_location="cpu")["model_state_dict"]
        model.load_state_dict({k[len("module."):] if k.startswith("module.") else k: v for k, v in ck.items()}, strict=False)
    return model.eval()


def main(args):
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model = load_model(args, dev)
    n = args.synthetic_rollout_steps or 100
    if args.num_envs > 1:
        wrapper = BatchedModelWrapper(model, args.num_envs, history_len=args.sequence_length,
                                      action_pred_steps=args.action_pred_steps, device=dev, incremental=args.incremental_rollout)
        lat = rollout_bench.run_batched(wrapper, n, "calvin", seed=args.seed, episode_len=360)
        rep = rollout_bench.batched_report(lat, min(2 * args.sequence_length + 5, n // 4), args.num_envs,
                                           "incremental" if args.incremental_rollout else "full_window")
        print(json.dumps({"metric": "batched_action_inference_latency_ms", **rep, "steps": n, "seq_len": args.sequence_length,
                          "wrapper": "calvin"}))
        return
    wrapper = ModelWrapper(model, history_len=args.sequence_length, action_pred_steps=args.action_pred_steps, device=dev,
                           incremental=args.incremental_rollout)
    lat = rollout_bench.run_calvin(wrapper, n, seed=args.seed, episode_len=360)          # EP_LEN of eval_utils_calvin.py:39
    rep = rollout_bench.percentile_report(lat, skip=min(2 * args.sequence_length + 5, n // 4))
    print(json.dumps({"metric": "action_inference_latency_ms", **rep, "steps": n, "seq_len": args.sequence_length,
                      "wrapper": "calvin", "incremental": bool(args.incremental_rollout)}))


if __name__ == "__main__":
    main(get_parser().parse_args())
