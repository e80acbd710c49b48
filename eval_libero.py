#!/usr/bin/env python
"""Entry point mirroring reference eval_libero.py:29-121: LIBERO action inference through the LIBERO rollout wrapper
(8-dim `--gripper_width` state or previous-gripper-command feedback, `--eval_libero_ensembling` temporal ensembling,
reference utils/eval_utils_libero.py:43-179).

The LIBERO simulator (MuJoCo / robosuite) is out of scope; `--synthetic_rollout_steps N` drives
`dreamvla_b200.utils.eval_utils_libero.ModelWrapper.step` with synthetic observations (agent-view and eye-in-hand images,
end-effector position + quaternion, finger joint positions) and reports p50 / p99 per-action latency.  A real env calls
`wrapper.step(...)` where the reference calls `model.step(obs, goal, steps)` (utils/eval_utils_libero.py:189).
The model is bf16 (`eval_calvin.load_model`); fp32 checkpoints load by rounding each value to bf16.
"""
from __future__ import annotations

import json

import torch

from dreamvla_b200.utils import rollout_bench
from dreamvla_b200.utils.arguments_utils import get_parser
from dreamvla_b200.utils.eval_utils_libero import ModelWrapper
from eval_calvin import load_model


def main(args):
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model = load_model(args, dev)
    wrapper = ModelWrapper(model, history_len=args.sequence_length, use_ensembling=args.eval_libero_ensembling,
                           ensembling_temp=args.ensembling_temp, libero_eval_max_steps=args.libero_eval_max_steps,
                           action_pred_steps=args.action_pred_steps, gripper_width=args.gripper_width, device=dev,
                           incremental=args.incremental_rollout)
    n = args.synthetic_rollout_steps or 100
    lat = rollout_bench.run_libero(wrapper, n, seed=args.seed, episode_len=args.libero_eval_max_steps)
    rep = rollout_bench.percentile_report(lat, skip=min(2 * args.sequence_length + 5, n // 4))
    print(json.dumps({"metric": "action_inference_latency_ms", **rep, "steps": n, "seq_len": args.sequence_length,
                      "wrapper": "libero", "gripper_width": bool(args.gripper_width),
                      "ensembling": bool(args.eval_libero_ensembling), "incremental": bool(args.incremental_rollout)}))


if __name__ == "__main__":
    main(get_parser().parse_args())
