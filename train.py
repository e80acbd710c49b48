#!/usr/bin/env python
"""Entry point mirroring reference train.py:40-297 for the H100-native hot path.

  torchrun --nnodes=1 --nproc_per_node=8 train.py <reference flags ...> [--synthetic_steps N] [--cuda_graph]

Builds `DreamVLA` from the reference's flags, casts to bf16 (`--precision bf16`; the kernels are bf16-only), sets up
one process per GPU over NCCL, and runs `train_one_epoch_calvin` (dreamvla_b200/utils/train_utils.py).  Dataset loading
(utils/data_utils.py in the reference) is out of scope: pass `--synthetic_steps N` to train on the synthetic collator
contract, or plug a loader that yields the reference's 13-tuple (data_utils.py:1395-1397) into `main(args, loader)`.
Checkpoints keep the reference's layout (train.py:279-289): {"epoch", "model_state_dict" ("module."-prefixed, trainable
parameters only; loadable by the reference and vice versa), "optimizer_state_dict", "lr_scheduler_state_dict"}.  The two
optimiser/scheduler entries are this package's own formats (flat fp32 AdamW moments keyed by parameter name; a step index)
and are restored on --resume_from_checkpoint; they are not interchangeable with torch.optim.AdamW / HF scheduler states.
"""
from __future__ import annotations

import math
import os
import random

import numpy as np
import torch

from dreamvla_b200 import ops
from dreamvla_b200.models import DreamVLA
from dreamvla_b200.utils.arguments_utils import get_parser, model_kwargs
from dreamvla_b200.utils.distributed_utils import init_distributed_device, world_info_from_env
from dreamvla_b200.utils.train_utils import StepConfig, TrainStep, synthetic_batch, train_one_epoch_calvin


def random_seed(seed=42, rank=0):           # train.py:23-26
    torch.manual_seed(seed + rank)
    np.random.seed(seed + rank)
    random.seed(seed + rank)
    ops.manual_seed(seed + rank)            # the kernels' Philox dropout stream follows --seed (and differs per rank)


class CosineRestartSchedule:
    """torch.optim.lr_scheduler.CosineAnnealingWarmRestarts(T_0=10, T_mult=2, eta_min=1e-7) stepped once per optimiser step
    with no epoch argument (train.py:205-206, train_utils.py:605): closed form of its T_cur / T_i recurrence."""

    def __init__(self, base_lr, T_0=10, T_mult=2, eta_min=1e-7):
        self.base_lr, self.T_0, self.T_mult, self.eta_min, self.step_idx = base_lr, T_0, T_mult, eta_min, 0

    def lr_at(self, s):
        T_i, t = self.T_0, s
        while t >= T_i:
            t -= T_i
            T_i *= self.T_mult
        return self.eta_min + (self.base_lr - self.eta_min) * (1 + math.cos(math.pi * t / T_i)) / 2

    def get_last_lr(self):
        return [self.lr_at(self.step_idx)]

    def step(self):
        self.step_idx += 1

    def state_dict(self):
        return {"step_idx": self.step_idx}

    def load_state_dict(self, sd):
        self.step_idx = sd["step_idx"]


class WarmupSchedule:
    """constant / linear / cosine with linear warm-up (transformers.get_*_schedule_with_warmup semantics, train.py:179-210)."""

    def __init__(self, base_lr, kind, warmup_steps, total_steps):
        self.base_lr, self.kind, self.warmup, self.total, self.step_idx = base_lr, kind, warmup_steps, max(total_steps, 1), 0

    def factor(self, s):
        if s < self.warmup:
            return s / max(1, self.warmup)
        if self.kind == "linear":
            return max(0.0, (self.total - s) / max(1, self.total - self.warmup))
        if self.kind == "cosine":
            prog = (s - self.warmup) / max(1, self.total - self.warmup)
            return max(0.0, 0.5 * (1.0 + math.cos(math.pi * prog)))
        return 1.0

    def get_last_lr(self):
        return [self.base_lr * self.factor(self.step_idx)]

    def step(self):
        self.step_idx += 1

    def state_dict(self):
        return {"step_idx": self.step_idx}

    def load_state_dict(self, sd):
        self.step_idx = sd["step_idx"]


class SyntheticLoader:
    """Yields the reference collator's 13-tuple (data_utils.py:1395-1397) from seeded synthetic tensors."""

    def __init__(self, args, device, steps):
        self.args, self.device, self.num_batches = args, device, steps
        self.cfg = StepConfig.from_args(args)

    def __iter__(self):
        a = self.args
        heads = dict(depth=a.depth_pred, dino=a.dino_feat_pred, sam=a.sam_feat_pred, traj=a.trajectory_pred, flow_mask=a.flow_as_mask)
        for i in range(self.num_batches):
            b = synthetic_batch(self.cfg, a.batch_size, "cpu", seed=a.seed + 1000 * a.rank + i, heads=heads, dtype=torch.float32)
            tracks = {"tracks": b["tracks"], "tracks_gripper": b["tracks_gripper"]} if "tracks" in b else {}
            yield (b["images_primary"], b["text"], b["actions"], b["images_wrist"], b["states"], None,
                   b.get("depth_primary"), b.get("depth_wrist"), b.get("dino_primary"), b.get("dino_wrist"),
                   b.get("sam_primary"), b.get("sam_wrist"), tracks)


class _ModuleWrapper:
    """`ddp_model.module` / "module."-prefixed state_dict surface of DistributedDataParallel (train.py:173,250,279-285);
    gradient averaging itself is the flat all-reduce inside TrainStep."""

    def __init__(self, module):
        self.module = module

    def train(self):
        self.module.train()

    def state_dict(self):
        return {"module." + k: v for k, v in self.module.state_dict().items()}

    def load_state_dict(self, sd, strict=False):
        return self.module.load_state_dict({k[len("module."):] if k.startswith("module.") else k: v for k, v in sd.items()}, strict=strict)

    def named_parameters(self):
        return (("module." + n, p) for n, p in self.module.named_parameters())


def get_checkpoint(model):                  # train_utils.py:750-757
    sd = model.state_dict()
    for name, p in model.named_parameters():
        if name in sd and not p.requires_grad:
            del sd[name]
    return sd


def main(args, loader=None):
    args.local_rank, args.rank, args.world_size = world_info_from_env()
    device_id = init_distributed_device(args)
    random_seed(args.seed)                   # train.py:50: every rank builds the SAME initial model
    if args.precision not in ("bf16", "amp_bf16", "amp_bfloat16"):
        raise SystemExit("dreamvla_b200 kernels are bf16-only: run with --precision bf16")
    model = DreamVLA(finetune_type=args.finetune_type, clip_device="cpu", vit_checkpoint_path=args.vit_checkpoint_path,
                     **model_kwargs(args))
    model = model.bfloat16()
    model.clip_model.requires_grad_(False)
    model.vision_encoder.requires_grad_(False)          # runs under no_grad in forward (dreamvla_model.py:670)
    model = model.to(device_id)
    model._init_model_type()
    ddp_model = _ModuleWrapper(model)
    random_seed(args.seed, args.rank)        # train.py:110: data order / dropout / diffusion draws differ per rank
    if loader is None:
        if args.synthetic_steps <= 0:
            raise SystemExit("dataset loading is out of scope of this package: pass --synthetic_steps N or call "
                             "main(args, loader) with a loader yielding the reference's 13-tuple batches")
        loader = SyntheticLoader(args, device_id, args.synthetic_steps)
    total_steps = loader.num_batches * args.num_epochs
    accum = max(args.gradient_accumulation_steps, 1)
    if args.lr_scheduler == "cosine_restart":
        sched = CosineRestartSchedule(args.learning_rate)
    else:                                    # train.py:179-210 (the "+ 1" only when accumulating)
        extra = 1 if accum > 1 else 0
        sched = WarmupSchedule(args.learning_rate, args.lr_scheduler, loader.num_batches * args.warmup_epochs // accum + extra,
                               total_steps // accum + extra)
    resume_from_epoch = 0
    if args.finetune_from_pretrained_ckpt is not None:   # train.py:212-250 key surgery
        ckpt = torch.load(args.finetune_from_pretrained_ckpt, map_location="cpu")["model_state_dict"]
        drop = []
        if args.reset_action_token: drop.append("module.action_pred_token")
        if args.reset_obs_token: drop.append("module.obs_tokens")
        if args.reset_mask_token: drop.append("module.mask_token")
        for k in list(ckpt):
            if (args.reset_image_decoder and "image_decoder" in k) or (args.reset_action_decoder and "action_decoder" in k) \
                    or (args.reset_resampler and "perceiver_resampler" in k) or k in drop:
                del ckpt[k]
        pe = "module.transformer_backbone_position_embedding"
        if pe in ckpt and ckpt[pe].shape != model.transformer_backbone_position_embedding.shape:
            ckpt[pe] = ckpt[pe][:, :args.sequence_length, :, :]
        ddp_model.load_state_dict(ckpt, False)
    opt_state = None
    if args.resume_from_checkpoint is not None:
        ck = torch.load(args.resume_from_checkpoint, map_location="cpu")
        ddp_model.load_state_dict(ck["model_state_dict"], False)
        opt_state = ck.get("optimizer_state_dict")
        sched.load_state_dict(ck["lr_scheduler_state_dict"])
        resume_from_epoch = ck["epoch"] + 1
    # The flat parameter / gradient / AdamW-moment buffers (the optimiser of this package) are built AFTER every checkpoint
    # load: parameters become views of one buffer, rank 0's copy is broadcast (DDP constructor semantics, train.py:173), and
    # a resumed run gets its moments and step count back (train.py:256).
    state = TrainStep(model, StepConfig.from_args(args), world_size=args.world_size)
    model._dvla_train_step = state
    if opt_state is not None:
        if opt_state.get("format") != "dvla_flat_adamw_v1":
            raise SystemExit("optimizer_state_dict is not in this package's flat-AdamW format (a torch.optim.AdamW state from "
                             "the reference cannot be mapped: it is index-keyed over a different parameter list)")
        state.flat.load_optimizer_state_dict(opt_state)
    ckpt_dir = os.path.join(f"{args.save_checkpoint_path}", args.run_name)
    if args.rank == 0 and args.save_checkpoint:
        os.makedirs(ckpt_dir, exist_ok=True)
    ddp_model.train()
    for epoch in range(resume_from_epoch, args.num_epochs):
        state = train_one_epoch_calvin(args=args, model=ddp_model, epoch=epoch, optimizer=None, lr_scheduler=sched,
                                       calvin_loader=loader, device_id=device_id, wandb=None)
        if args.rank == 0 and args.save_checkpoint and epoch % args.save_checkpoint_seq == 0 and epoch > args.start_save_checkpoint:
            torch.save({"epoch": epoch, "model_state_dict": get_checkpoint(ddp_model),
                        "optimizer_state_dict": state.flat.optimizer_state_dict(),
                        "lr_scheduler_state_dict": sched.state_dict()}, os.path.join(ckpt_dir, f"{epoch}.pth"))
    if args.rank == 0 and state is not None:
        print(f"[train] done: {state.total_micro} micro-steps, last loss terms "
              f"{ {k: round(float(v), 5) for k, v in state.last_terms.items()} }")
    return state


if __name__ == "__main__":
    main(get_parser().parse_args())          # the returned state (and with it any captured graphs) is dropped here
    from dreamvla_b200.utils.distributed_utils import shutdown_distributed
    shutdown_distributed()
