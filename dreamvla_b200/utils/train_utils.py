"""Train step of the hot path -- H100-native mirror of reference utils/train_utils.py:59-726 (`train_one_epoch_calvin`).

Reference step (train_utils.py:94-608): unpack the 13-tuple batch, build labels, forward, seven losses with weights
(1.0 arm, 0.01 gripper, 0.1 image, 0.001 depth, 0.1 traj(x0.1), 0.01 dino, 0.01 sam, :585), `/accum`, backward (DDP
all-reduce), clip_grad_norm_(0.1) every micro-step, AdamW / scheduler / zero_grad on accumulation boundaries.

Here:
  * FlatParams keeps parameters, gradients and AdamW moments in flat buffers; weight gradients are accumulated straight
    into the flat gradient buffer by the wgrad GEMM epilogue (ops.py), 1-D gradients in an fp32 side buffer;
  * losses are fused value+gradient kernels (ops.mse_loss / cosine_loss / silog_loss), no host sync in the step;
  * data-parallel: the flat bf16 gradient buffer is laid out in order of backward completion and all-reduced (NCCL over
    NVLink, communication stream) in three segments, the first two from backward hooks while backward continues; then
    an order-deterministic global norm + clip + AdamW in two kernels (dvla_sumsq, dvla_adamw; dvla_adamw_master on fp32
    master weights under --precision fp32); lr / step counters live on the device;
  * the per-step `.cpu().numpy()` visual-debug copies of the reference (:198-213, :382-396) are not part of the path.
"""
from __future__ import annotations

import math
import os
import re
import time
from dataclasses import dataclass

import torch
import torch.nn.functional as F

from .. import _lib as L
from .. import ops

# parameters that exist in the reference's module tree but never receive a gradient in forward (dreamvla_model.py:
# 203-205 action encoders, :320-333 recon_* decoders, action_model/models.py:187 history_embedder; the frozen ViT/CLIP).
NEVER_USED_PREFIXES = ("vision_encoder.", "clip_model.", "recon_state_decoder.", "recon_arm_state_decoder.",
                       "recon_gripper_state_decoder.", "action_pose_encoder.", "action_gripper_position_encoder.",
                       "action_projector.", "action_model.net.history_embedder.")
HEAD_PREFIXES = {
    "image": ("image_decoder", "mask_token", "obs_tokens"),
    "depth": ("depth_decoder", "depth_mask_token", "depth_tokens"),
    "dino": ("dino_feat_decoder", "dino_decoder", "dino_mask_token", "dino_feat_tokens"),
    "sam": ("sam_feat_decoder", "sam_decoder", "sam_mask_token", "sam_feat_tokens"),
    "traj": ("traj_decoder", "traj_mask_token", "trajectory_tokens"),
}


# Parameters whose gradients are complete once the backward pass reaches the backbone output (decoders, heads, DiT): their
# flat-buffer segment is all-reduced while the backbone is still back-propagating.  (The query tokens `obs_tokens`,
# `*_tokens`, `action_pred_token` are INPUTS of the backbone: their gradients complete last.)
EARLY_GRAD_PREFIXES = ("image_decoder", "mask_token", "depth_decoder", "depth_mask_token", "dino_feat_decoder", "dino_decoder",
                       "dino_mask_token", "sam_feat_decoder", "sam_decoder", "sam_mask_token", "traj_decoder", "traj_mask_token",
                       "action_model.", "action_decoder", "arm_action_decoder", "gripper_action_decoder")


BACKBONE_CUTS = 3          # the backbone's gradients are exchanged in BACKBONE_CUTS + 1 pieces (layer quarters at 3)


def backbone_cut_layers(n_layers: int, n_cuts: int = BACKBONE_CUTS):
    """Layer indices (descending) at whose INPUT a gradient segment completes during backward: with 24 layers and 3 cuts
    [18, 12, 6] -- the gradients of layers >= 18 are final once backward reaches the input of layer 18, and so on."""
    n_cuts = max(0, min(n_cuts, n_layers - 1))
    return sorted({max(1, round(n_layers * (n_cuts - i) / (n_cuts + 1))) for i in range(n_cuts)}, reverse=True)


def grad_segment(name: str, n_layers: int, n_cuts: int = BACKBONE_CUTS) -> int:
    """Order in which a parameter's gradient becomes final during backward.  0: complete when backward reaches the backbone
    output (heads, decoders, DiT); k = 1..len(cuts): backbone layers >= cuts[k-1] (and `ln_f` with k = 1), complete at the
    input of layer cuts[k-1]; len(cuts) + 1: everything that feeds the backbone -- complete only at the end."""
    if name.startswith(EARLY_GRAD_PREFIXES):
        return 0
    cuts = backbone_cut_layers(n_layers, n_cuts)
    if name.startswith("transformer_backbone.ln_f."):
        return 1 if cuts else len(cuts) + 1
    m = re.match(r"transformer_backbone\.h\.(\d+)\.", name)
    if m:
        layer = int(m.group(1))
        for k, c in enumerate(cuts):
            if layer >= c:
                return k + 1
    return len(cuts) + 1


def get_cast_dtype(precision: str):
    """train_utils.py:16-22."""
    if precision in ("bf16", "amp_bf16", "amp_bfloat16"):
        return torch.bfloat16
    if precision == "fp16":
        return torch.float16
    return None


class AverageMeter:
    """train_utils.py:764-780."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.val = self.avg = self.sum = self.count = 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


def patchify(imgs, patch_size):
    """train_utils.py:37-50."""
    h = w = imgs.shape[2] // patch_size
    x = imgs.reshape(imgs.shape[0], 3, h, patch_size, w, patch_size)
    x = torch.einsum("nchpwq->nhwpqc", x)
    return x.reshape(imgs.shape[0], h * w, patch_size ** 2 * 3)


def normalize_patchfied_image(x):
    """train_utils.py:52-57 (unbiased variance, eps 1e-6)."""
    mean = x.mean(dim=-1, keepdim=True)
    var = x.var(dim=-1, keepdim=True)
    return (x - mean) / (var + 1.0e-6) ** 0.5


def unpatchify(patches, patch_size=16, img_size=(224, 224)):
    """train_utils.py:783-799."""
    B, P, n, pd = patches.shape
    g = int(n ** 0.5)
    C = pd // (patch_size * patch_size)
    x = patches.view(B, P, g, g, patch_size, patch_size, C).permute(0, 1, 6, 2, 4, 3, 5).contiguous()
    return x.view(B, P, C, *img_size)


def patchify_map(img, patch_size=16):
    """Inverse of `unpatchify` for C = 1 maps: [n, 1, H, W] -> [n, (H/p)(W/p), p*p].  SiLog is a mean over elements, so
    permuting the LABEL instead of un-permuting the prediction (train_utils.py:366-371) gives the identical loss."""
    n, _, H, W = img.shape
    g = H // patch_size
    return img.view(n, g, patch_size, g, patch_size).permute(0, 1, 3, 2, 4).reshape(n, g * g, patch_size * patch_size)


def flow_masks(tracks_primary, tracks_wrist):
    """train_utils.py:274-313: 28x28 flow -> avg-pool 2x2 -> |v| > 1 -> (primary only) 3x3 max-pool dilation.
    Returns per-patch {0,1} masks [n*196] for each camera."""
    Bn, P, HW, C = tracks_primary.shape
    H = W = int(HW ** 0.5)

    def pool(t):
        tp = t.reshape(Bn * P, H, W, C).permute(0, 3, 1, 2).float()
        return (torch.norm(F.avg_pool2d(tp, kernel_size=2, stride=2), dim=1) > 1.0).unsqueeze(1).float()
    mp = F.max_pool2d(pool(tracks_primary), kernel_size=3, stride=1, padding=1)
    mw = pool(tracks_wrist)
    return mp.reshape(-1).contiguous(), mw.reshape(-1).contiguous()


@dataclass
class StepConfig:
    sequence_length: int = 10
    future_steps: int = 3
    action_pred_steps: int = 3
    atten_goal: int = 0
    pred_num: int = 1
    patch_size: int = 16
    use_dit_head: bool = True
    loss_action: bool = True
    loss_image: bool = False
    loss_depth: bool = False
    loss_dino_feat: bool = False
    loss_sam_feat: bool = False
    loss_trajectory: bool = False
    flow_as_mask: bool = False
    loss_arm_action_ratio: float = 1.0
    loss_gripper_action_ratio: float = 0.01
    gradient_accumulation_steps: int = 1
    learning_rate: float = 1e-3
    weight_decay: float = 1e-4
    max_grad_norm: float = 0.1
    gripper_width: bool = False
    # True (reference semantics, utils/train_utils.py:599-600 + DDP without no_sync): the gradient is all-reduced and the
    # ACCUMULATED gradient is clipped in place after EVERY micro-step.  False: one exchange + one clip per optimiser step
    # (cheaper, but a different update whenever gradient_accumulation_steps > 1).
    reduce_every_micro_step: bool = True

    @staticmethod
    def from_args(args):
        kw = {f: getattr(args, f) for f in StepConfig.__dataclass_fields__ if hasattr(args, f)}
        if getattr(args, "exchange_on_boundary_only", False):
            kw["reduce_every_micro_step"] = False
        return StepConfig(**kw)


class FlatParams:
    """Flat bf16 parameter / gradient buffers + fp32 AdamW moments for the trainable, USED parameters of a DreamVLA.

    Layout: [ >=2-D parameters | 1-D parameters ], each parameter 16-byte aligned.  Parameters become views of `P`;
    `p.grad` is a view of `G`; ops accumulate weight gradients through `p._dvla_grad` and 1-D gradients in fp32
    through `p._dvla_grad32` (folded into G by `fold_small_grads`).

    `master` (`--precision fp32`): a dict name -> fp32 tensor with the fp32 values of (at least) the trainable parameters.
    Then `P32` holds fp32 master weights in the same layout as `P`, AdamW updates `P32` (dvla_adamw_master) and `P` is
    the bf16 working copy, rounded from `P32` once per optimiser step.  Without it `P32` is None and AdamW updates `P`."""

    def __init__(self, model, cfg: StepConfig, exclude_prefixes=(), master=None):
        inactive = []
        for head, on in (("image", cfg.loss_image), ("depth", cfg.loss_depth), ("dino", cfg.loss_dino_feat),
                         ("sam", cfg.loss_sam_feat), ("traj", cfg.loss_trajectory)):
            if not on:
                inactive += list(HEAD_PREFIXES[head])
        skip = tuple(NEVER_USED_PREFIXES) + tuple(exclude_prefixes)
        big, small = [], []
        self.names = []
        for name, p in model.named_parameters():
            if not p.requires_grad or name.startswith(skip) or any(name.startswith(pref) for pref in inactive):
                continue
            if not model.use_dit_head and name.startswith("action_model."):
                continue
            if p.dtype != torch.bfloat16 or not p.is_cuda:
                raise RuntimeError(f"FlatParams: {name} is {p.dtype} on {p.device}; the train step is bf16/CUDA only")
            (small if p.dim() <= 1 else big).append((name, p))
        n_layers = len(model.transformer_backbone.h)
        big.sort(key=lambda np_: grad_segment(np_[0], n_layers))          # stable: registration order inside a segment
        self.params = big + small
        dev = self.params[0][1].device

        def aligned(n):
            return (n + 7) // 8 * 8
        off = 0
        offs = []
        for _, p in self.params:
            offs.append(off)
            off += aligned(p.numel())
        self.n_big = sum(aligned(p.numel()) for _, p in big)
        self.n = off
        # [0, seg_end[0]), [seg_end[0], seg_end[1]), ... hold the >=2-D gradients of segments 0, 1, ... (see grad_segment);
        # the last segment (and the 1-D gradients behind it) is complete only when backward has finished
        self.cut_layers = backbone_cut_layers(n_layers)
        self.seg_end = [sum(aligned(p.numel()) for n_, p in big if grad_segment(n_, n_layers) <= k)
                        for k in range(len(self.cut_layers) + 1)]
        self.P = torch.zeros(self.n, device=dev, dtype=torch.bfloat16)
        self.G = torch.zeros(self.n, device=dev, dtype=torch.bfloat16)
        self.G32 = torch.zeros(max(self.n - self.n_big, 8), device=dev, dtype=torch.float32)
        self.m = torch.zeros(self.n, device=dev, dtype=torch.float32)
        self.v = torch.zeros(self.n, device=dev, dtype=torch.float32)
        self.sumsq = torch.zeros(1, device=dev, dtype=torch.float32)
        self.lr = torch.zeros(1, device=dev, dtype=torch.float32)
        self.step_count = torch.zeros(1, device=dev, dtype=torch.float32)
        self.P32 = None
        if master is not None:
            self.P32 = torch.zeros(self.n, device=dev, dtype=torch.float32)
            for (name, p), o in zip(self.params, offs):
                if name not in master or master[name].shape != p.shape:
                    raise RuntimeError(f"FlatParams: no fp32 master value of shape {tuple(p.shape)} for {name}")
                self.P32[o:o + p.numel()].copy_(master[name].reshape(-1))
            self.P.copy_(self.P32)
        for (name, p), o in zip(self.params, offs):
            n = p.numel()
            if self.P32 is None:
                self.P[o:o + n].copy_(p.data.reshape(-1))
            p.data = self.P[o:o + n].view(p.shape)
            g = self.G[o:o + n].view(p.shape)
            p.grad = g
            p._dvla_grad = g
            if p.dim() <= 1:
                p._dvla_grad32 = self.G32[o - self.n_big:o - self.n_big + n]
            self.names.append(name)
        self.offsets = offs
        self.num_params = sum(p.numel() for _, p in self.params)
        # fp32 values of the trainable parameters this step never updates (NEVER_USED_PREFIXES, heads whose loss is off),
        # kept on the host so that a checkpoint writes back exactly what was loaded
        trained = set(self.names)
        self.master_rest = {} if master is None else {
            name: master[name].detach().to("cpu", torch.float32).clone() for name, p in model.named_parameters()
            if p.requires_grad and name not in trained and name in master}

    def master_state_dict(self):
        """name -> fp32 value of every trainable parameter in fp32 mode: views of `P32` for the parameters the step trains,
        then the host copies of `master_rest`."""
        sd = {name: self.P32[o:o + p.numel()].view(p.shape) for (name, p), o in zip(self.params, self.offsets)}
        sd.update(self.master_rest)
        return sd

    def fold_small_grads(self):
        if self.n > self.n_big:
            L.accum_fp32_into_bf16(self.G32[: self.n - self.n_big], self.G[self.n_big:])
            self.G32.zero_()

    def clip_in_place(self, cfg: StepConfig, world_size: int = 1):
        """G <- clip_grad_norm_(G / world, max_norm) in the buffer itself: what the reference does to the accumulated .grad
        after every micro-step (train_utils.py:599-600); G holds the rank SUM when this is called."""
        self.sumsq.zero_()
        L.sumsq(self.G, self.sumsq)
        L.grad_clip_scale(self.G, self.sumsq, cfg.max_grad_norm, 1.0 / world_size)

    def optimizer_step(self, cfg: StepConfig, lr: float | None, world_size: int = 1, preclipped: bool = False):
        """clip_grad_norm_(max_norm) on the rank-averaged gradient + AdamW (train_utils.py:600-608); zeroes G.
        lr=None keeps the device-resident lr (set outside a captured CUDA graph).  preclipped=True: G already holds the
        rank mean, clipped by `clip_in_place` (gradient accumulation with the reference's per-micro-step clip)."""
        if lr is not None:
            self.lr.fill_(lr)
        self.step_count += 1
        if self.P32 is None:
            def update(**kw):
                L.adamw(self.P, self.G, self.m, self.v, **kw)
        else:
            def update(**kw):
                L.adamw_master(self.P32, self.P, self.G, self.m, self.v, **kw)
        if preclipped:
            update(sumsq_t=None, lr_t=self.lr, step_t=self.step_count, beta1=0.9, beta2=0.999, eps=1e-8,
                   weight_decay=cfg.weight_decay, max_norm=cfg.max_grad_norm, grad_scale=1.0, zero_grad=True)
            return
        self.sumsq.zero_()
        L.sumsq(self.G, self.sumsq)
        update(sumsq_t=self.sumsq, lr_t=self.lr, step_t=self.step_count, beta1=0.9, beta2=0.999, eps=1e-8,
               weight_decay=cfg.weight_decay, max_norm=cfg.max_grad_norm, grad_scale=1.0 / world_size, zero_grad=True)

    def optimizer_state_dict(self):
        """AdamW state of the flat buffers.  NOT torch.optim.AdamW's format (the reference's `optimizer_state_dict`,
        train.py:283, is index-keyed over its own parameter list and holds bf16 moments): moments here are fp32 and keyed by
        the parameter names in `names`, in flat-buffer order."""
        return {"format": "dvla_flat_adamw_v1", "names": list(self.names), "numel": [p.numel() for _, p in self.params],
                "m": self.m.detach().cpu(), "v": self.v.detach().cpu(), "step": self.step_count.detach().cpu()}

    def load_optimizer_state_dict(self, sd):
        if sd.get("names") != list(self.names) or tuple(sd["m"].shape) != tuple(self.m.shape):
            raise RuntimeError("optimizer state does not match this model's trainable parameter set "
                               "(saved by a different head configuration?)")
        self.m.copy_(sd["m"])
        self.v.copy_(sd["v"])
        self.step_count.copy_(sd["step"].reshape(-1)[:1])


def build_labels(cfg: StepConfig, batch, need):
    """Label tensors for the enabled losses (train_utils.py:171-185, 340-342, 400-402, 429-431, 455-477), bf16, on device.
    `batch` is a dict (see synthetic_batch); windows are [B, W, ...] with W = sequence_length + future_steps."""
    S, fs = cfg.sequence_length, cfg.future_steps
    n_lab = S - cfg.atten_goal
    out = {}
    with torch.no_grad():
        if need.get("image"):
            for cam, key in (("p", "images_primary"), ("w", "images_wrist")):
                lab = batch[key][:, fs:fs + n_lab].flatten(0, 1).float()
                out["image_" + cam] = normalize_patchfied_image(patchify(lab, cfg.patch_size)).to(torch.bfloat16).contiguous()
            if cfg.flow_as_mask and "tracks" in batch:
                out["mask_p"], out["mask_w"] = flow_masks(batch["tracks"][:, :n_lab], batch["tracks_gripper"][:, :n_lab])
        if need.get("depth"):
            for cam, key in (("p", "depth_primary"), ("w", "depth_wrist")):
                lab = batch[key][:, fs:fs + n_lab].flatten(0, 1)
                out["depth_" + cam] = patchify_map(lab, cfg.patch_size).to(torch.bfloat16).contiguous()
        if need.get("dino"):
            out["dino_p"] = batch["dino_primary"][:, fs:fs + n_lab].flatten(0, 1).to(torch.bfloat16).contiguous()
            out["dino_w"] = batch["dino_wrist"][:, fs:fs + n_lab].flatten(0, 1).to(torch.bfloat16).contiguous()
        if need.get("sam"):
            out["sam_p"] = batch["sam_primary"][:, fs:fs + n_lab].flatten(0, 1).to(torch.bfloat16).contiguous()
            out["sam_w"] = batch["sam_wrist"][:, fs:fs + n_lab].flatten(0, 1).to(torch.bfloat16).contiguous()
        if need.get("traj"):
            for cam, key in (("p", "tracks"), ("w", "tracks_gripper")):
                t = batch[key][:, :n_lab]
                h = w = int(math.sqrt(t.shape[-2]))
                t = t.reshape(t.shape[0], t.shape[1], h, w, t.shape[-1]).permute(0, 1, 4, 2, 3)
                t = F.pixel_unshuffle(t, downscale_factor=h // 14)
                out["traj_" + cam] = t.flatten(3).permute(0, 1, 3, 2).flatten(0, 1).to(torch.bfloat16).contiguous()
    return out


def compute_losses(cfg: StepConfig, outputs, labels, bs, unit_upstream=True):
    """Weighted loss terms of train_utils.py:158-170,325-337,366-371,423-425,448-450,499-502,585 as fused kernels.
    Every returned tensor already carries its weight of the total (:585) and 1/accum (:588)."""
    (arm, gripper, image_pred, _, _, _, depth_pred, traj_pred, dino_pred, sam_pred) = outputs
    S = cfg.sequence_length
    n_lab = S - cfg.atten_goal
    acc = 1.0 / cfg.gradient_accumulation_steps
    terms = {}

    def trim(t):   # [B*S, 2, P, N, C] -> first S - atten_goal timesteps (train_utils.py:187-189)
        if n_lab == S:
            return t
        return t.reshape(bs, S, *t.shape[1:])[:, :n_lab].reshape(-1, *t.shape[1:])

    if cfg.use_dit_head:
        terms["action"] = arm * (cfg.loss_arm_action_ratio * acc)
    elif cfg.loss_action and cfg.action_pred_steps:
        la = labels["actions"]
        terms["arm"] = F.smooth_l1_loss(arm[:, :n_lab].float(), la[..., :6].float()) * (cfg.loss_arm_action_ratio * acc)
        terms["gripper"] = F.binary_cross_entropy(gripper[:, :n_lab].float(), la[..., 6:].float()) * (cfg.loss_gripper_action_ratio * acc)
    if cfg.loss_image and image_pred is not None:
        ip = trim(image_pred)
        w = 0.1 * 0.5 * acc
        terms["image"] = (ops.mse_loss(ip[:, 0, 0], labels["image_p"], labels.get("mask_p"), w, unit_upstream)
                          + ops.mse_loss(ip[:, 1, 0], labels["image_w"], labels.get("mask_w"), w, unit_upstream))
    if cfg.loss_depth and depth_pred is not None:
        dp = trim(depth_pred)
        w = 0.001 * 0.5 * acc
        terms["depth"] = (ops.silog_loss(dp[:, 0, 0], labels["depth_p"], 0.5, w, unit_upstream)
                          + ops.silog_loss(dp[:, 1, 0], labels["depth_w"], 0.5, w, unit_upstream))
    if cfg.loss_dino_feat and dino_pred is not None:
        dp = trim(dino_pred)
        w = 0.01 * 0.5 * acc
        terms["dino"] = (ops.cosine_loss(dp[:, 0, 0], labels["dino_p"], w, unit_upstream)
                         + ops.cosine_loss(dp[:, 1, 0], labels["dino_w"], w, unit_upstream))
    if cfg.loss_sam_feat and sam_pred is not None:
        sp = trim(sam_pred)
        w = 0.01 * 0.5 * acc
        terms["sam"] = (ops.cosine_loss(sp[:, 0, 0], labels["sam_p"], w, unit_upstream)
                        + ops.cosine_loss(sp[:, 1, 0], labels["sam_w"], w, unit_upstream))
    if cfg.loss_trajectory and traj_pred is not None:
        tp = trim(traj_pred)
        w = 0.1 * 0.1 * acc
        terms["traj"] = (ops.mse_loss(tp[:, 0, 0], labels["traj_p"], None, w, unit_upstream)
                         + ops.mse_loss(tp[:, 1, 0], labels["traj_w"], None, w, unit_upstream))
    return terms


def all_reduce_flat(G, world_size, group=None, comm_stream=None):
    """SUM all-reduce of the flat gradient buffer (the 1/world of DDP's mean is applied later as `grad_scale` inside the
    clip+AdamW kernel).  On CUDA it runs on `comm_stream`, ordered after the producer stream and before its consumers."""
    if world_size == 1:
        return
    import torch.distributed as dist
    if comm_stream is None or not G.is_cuda:
        dist.all_reduce(G, op=dist.ReduceOp.SUM, group=group)
        return
    cur = torch.cuda.current_stream()
    comm_stream.wait_stream(cur)
    with torch.cuda.stream(comm_stream):
        dist.all_reduce(G, op=dist.ReduceOp.SUM, group=group)
    cur.wait_stream(comm_stream)


class TrainStep:
    """One micro-step of train_utils.py:94-608 on device-resident inputs; see module docstring."""

    def __init__(self, model, cfg: StepConfig, world_size=1, process_group=None, master=None):
        """`master`: fp32 values of the trainable parameters (name -> tensor) for fp32 master weights, see FlatParams."""
        if cfg.pred_num != 1:
            # the reference unfolds the labels over pred_num (train_utils.py:176-185); this step builds single-frame labels
            raise NotImplementedError("pred_num > 1 is not implemented in the train step (labels are not unfolded)")
        self.model, self.cfg = model, cfg
        self.world_size = world_size
        self.pg = process_group
        self.flat = FlatParams(model, cfg, master=master)
        if world_size > 1:
            # DDP's constructor broadcasts rank 0's parameters and buffers (train.py:173); every replica must start from
            # the same weights or the shared all-reduced gradient is applied to different models
            import torch.distributed as dist
            if self.flat.P32 is not None:
                dist.broadcast(self.flat.P32, src=0, group=process_group)
                self.flat.P.copy_(self.flat.P32)
            else:
                dist.broadcast(self.flat.P, src=0, group=process_group)
            for _, b in model.named_buffers():
                if b.is_cuda:
                    dist.broadcast(b, src=0, group=process_group)
            for name, p in model.named_parameters():
                if p.is_cuda and not name.startswith("clip_model.") and getattr(p, "_dvla_grad", None) is None:
                    dist.broadcast(p.data, src=0, group=process_group)
        self.micro = 0            # position inside the current accumulation window
        self.total_micro = 0      # micro-steps since construction
        self.comm_stream = torch.cuda.Stream() if world_size > 1 else None
        self.last_terms = {}
        # The gradient segments that complete early (heads/decoders/DiT, then the second half of the backbone) are all-reduced
        # from backward hooks on the communication stream, overlapping the rest of the backward pass; the remainder follows
        # after backward.  tools/ddp_overlap_check.py compares it on 2 GPUs against one flat all-reduce, eagerly and inside the
        # captured step.  DVLA_AR_OVERLAP=0 turns it off.
        self.overlap = world_size > 1 and os.environ.get("DVLA_AR_OVERLAP", "1") != "0"
        self._reduced_upto = 0
        # while gradient segments are in flight the persistent GEMMs of backward are sized for the SMs NCCL leaves free
        # (DVLA_SM_BUDGET=0 turns that off)
        from .distributed_utils import nccl_cta_budget
        self.comm_ctas = nccl_cta_budget() if (self.overlap and os.environ.get("DVLA_SM_BUDGET", "1") != "0") else 0

    def prepare_inputs(self, batch):
        """train_utils.py:99-145: slices of the window, gripper remap, sliding-window action labels."""
        cfg = self.cfg
        S = cfg.sequence_length
        states = batch["states"]
        if cfg.gripper_width:
            input_states = torch.cat([states[..., :6], states[..., -2:]], dim=-1)
        else:
            input_states = torch.cat([states[..., :6], states[..., -1:]], dim=-1)
            input_states[..., 6:] = torch.div(input_states[..., 6:] + 1, 2, rounding_mode="floor")
        actions = batch["actions"].clone()
        actions[..., 6:] = torch.div(actions[..., 6:] + 1, 2, rounding_mode="floor")
        label_actions = torch.cat([actions[:, j:S - cfg.atten_goal + j, :].unsqueeze(-2)
                                   for j in range(cfg.action_pred_steps)], dim=-2)
        text = batch["text"].unsqueeze(1).expand(-1, S, -1)
        return dict(image_primary=batch["images_primary"][:, :S], image_wrist=batch["images_wrist"][:, :S],
                    state=input_states[:, :S], text_token=text, action_label=label_actions[:, :S - cfg.atten_goal])

    def forward_backward(self, batch, draws=None):
        """`draws` (tests): {"diffusion_noise", "diffusion_timestep", "diffusion_drop_ids"} -- the tensors the DiT loss samples
        (action_model.py:59-60, models.py:83), injected so a run can be lined up with the reference's recorded draws."""
        cfg = self.cfg
        inp = self.prepare_inputs(batch)
        need = dict(image=cfg.loss_image, depth=cfg.loss_depth, dino=cfg.loss_dino_feat, sam=cfg.loss_sam_feat,
                    traj=cfg.loss_trajectory)
        labels = build_labels(cfg, batch, need)
        labels["actions"] = inp["action_label"]
        outputs = self.model(inp["image_primary"], inp["image_wrist"], inp["state"], inp["text_token"], action=None,
                             action_label=inp["action_label"], **(draws or {}))
        terms = compute_losses(cfg, outputs, labels, bs=inp["state"].shape[0])
        total = None
        for t in terms.values():
            total = t if total is None else total + t
        total.backward()
        self.flat.fold_small_grads()
        self.last_terms = {k: v.detach() for k, v in terms.items()}
        return total.detach()

    def _reduce_segment(self, k):
        """Backward-pass hook: flat-gradient segment k is complete on the compute stream -> SUM all-reduce it on the
        communication stream (NCCL over NVLink) while the backward pass goes on."""
        import torch.distributed as dist
        lo, hi = self._reduced_upto, self.flat.seg_end[k]
        if hi <= lo:
            return
        ev = torch.cuda.current_stream().record_event()
        self.comm_stream.wait_event(ev)
        with torch.cuda.stream(self.comm_stream):
            dist.all_reduce(self.flat.G[lo:hi], op=dist.ReduceOp.SUM, group=self.pg)
        self._reduced_upto = hi
        if self.comm_ctas:
            L.set_sm_budget(torch.cuda.get_device_properties(self.flat.G.device).multi_processor_count - self.comm_ctas)

    def _arm_overlap(self):
        self._reduced_upto = 0
        if self.overlap:
            self.model._dvla_grad_marks = {
                "backbone_out": lambda: self._reduce_segment(0),
                "backbone_cuts": [(layer, (lambda k=k: self._reduce_segment(k + 1))) for k, layer in enumerate(self.flat.cut_layers)]}
        elif hasattr(self.model, "_dvla_grad_marks"):
            self.model._dvla_grad_marks = None

    def all_reduce_grads(self):
        """DDP gradient mean (train.py:173) as SUM all-reduces of the flat bf16 gradient buffer over NCCL on a side stream
        (the 1/world factor is applied inside the clip+AdamW kernel): the segments reduced by the backward hooks, then the
        rest here."""
        if self.world_size == 1:
            return
        lo = self._reduced_upto
        if self.comm_ctas:
            L.set_sm_budget(0)               # backward is over: the optimiser kernels wait for the exchange anyway
        all_reduce_flat(self.flat.G[lo:] if lo else self.flat.G, self.world_size, self.pg, self.comm_stream)
        self._reduced_upto = 0

    @property
    def per_micro_clip(self):
        """Reference accumulation semantics: reduce + clip the accumulated gradient in place after every micro-step."""
        return self.cfg.reduce_every_micro_step and self.cfg.gradient_accumulation_steps > 1

    def is_boundary(self, boundary=None):
        return ((self.micro + 1) % self.cfg.gradient_accumulation_steps == 0) if boundary is None else bool(boundary)

    def __call__(self, batch, lr=None, boundary=None, draws=None):
        """Micro-step: returns the (device) loss.  The reference all-reduces (DDP, no no_sync) and clips the accumulated
        gradient EVERY micro-step and steps the optimiser on accumulation boundaries and on the last batch of an epoch
        (train_utils.py:599-608); `boundary` overrides the internal counter for that last-batch case."""
        cfg = self.cfg
        self.flat.lr.fill_(cfg.learning_rate if lr is None else lr)
        b = self.is_boundary(boundary)
        loss = self.micro_step(batch, boundary=b, draws=draws)
        self.micro += 1
        self.total_micro += 1
        if b:
            self.flat.optimizer_step(cfg, None, self.world_size, preclipped=self.per_micro_clip)
            self.micro = 0
        return loss

    def micro_step(self, batch, boundary=None, draws=None):
        ops.seed_counter(self.flat.P.device).add_(1)        # fresh dropout masks every step, also under graph replay
        boundary = self.is_boundary(boundary)
        # reference semantics: exchange every micro-step; otherwise only on accumulation boundaries (same mean, one clip)
        exchange = boundary or self.cfg.reduce_every_micro_step
        if exchange:
            self._arm_overlap()
        elif hasattr(self.model, "_dvla_grad_marks"):
            self.model._dvla_grad_marks = None
        try:
            loss = self.forward_backward(batch, draws)
        finally:
            if getattr(self.model, "_dvla_grad_marks", None) is not None:
                self.model._dvla_grad_marks = None       # a bare forward_backward() outside the step must never reduce
            if self.comm_ctas:
                L.set_sm_budget(0)
        if exchange:
            self.all_reduce_grads()
        if self.per_micro_clip:
            self.flat.clip_in_place(self.cfg, self.world_size)
        return loss


class GraphedTrainStep:
    """The whole micro-step (forward, losses, backward, all-reduce) and the optimiser step captured as two CUDA graphs:
    the reference issues ~4-5 k kernel launches per step from Python; a replay is one launch.  Inputs are copied into
    static device buffers (that copy IS the H2D transfer when the source is pinned host memory)."""

    def __init__(self, step: TrainStep, example_batch, warmup=3):
        if step.world_size > 1 and step.cfg.gradient_accumulation_steps != 1 and not step.cfg.reduce_every_micro_step:
            raise ValueError("GraphedTrainStep: the captured micro-step contains the gradient all-reduce; with "
                             "reduce_every_micro_step=False and world_size > 1 use gradient_accumulation_steps == 1 or the "
                             "eager TrainStep")
        self.step = step
        self.static = {k: v.clone() for k, v in example_batch.items()}
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):                       # real steps: allocator pools, caches, lazy tables
                step(self.static)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        n0 = L.launch_count()
        self.g_micro = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g_micro):
            # with the reference's accumulation semantics every micro-step is the same graph (exchange + in-place clip);
            # without accumulation it is the boundary step
            self.loss = step.micro_step(self.static, boundary=step.cfg.gradient_accumulation_steps == 1 or None)
        self.g_opt = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g_opt, pool=self.g_micro.pool()):
            step.flat.optimizer_step(step.cfg, None, step.world_size, preclipped=step.per_micro_clip)
        self.launches_per_step = L.launch_count() - n0      # libdvla kernels recorded in the two graphs

    def __call__(self, batch, lr=None, boundary=None):
        st = self.step
        if batch is not self.static:
            for k, v in batch.items():
                self.static[k].copy_(v, non_blocking=True)
        if lr is not None:
            st.flat.lr.fill_(lr)
        b = st.is_boundary(boundary)
        self.g_micro.replay()
        st.micro += 1
        st.total_micro += 1
        if b:
            self.g_opt.replay()
            st.micro = 0
        return self.loss


def synthetic_batch(cfg: StepConfig, batch_size, device, seed=1234, heads=None, dtype=torch.bfloat16, pin=False):
    """Synthetic batch with the collator's output contract (data_utils.py:1395-1397; SURVEY §8d), seeded.
    Returned as a dict of tensors on `device` (or pinned host tensors with pin=True)."""
    heads = heads or {}
    W = cfg.sequence_length + cfg.future_steps
    g = torch.Generator(device="cpu").manual_seed(seed)
    B = batch_size

    def rn(*shape, scale=1.0):
        return (torch.randn(*shape, generator=g) * scale)
    text = torch.zeros(B, 77, dtype=torch.int32)
    for b in range(B):
        k = int(torch.randint(3, 21, (1,), generator=g))
        text[b, 0] = 49406
        text[b, 1:1 + k] = torch.randint(1, 49406, (k,), generator=g, dtype=torch.int32)
        text[b, 1 + k] = 49407
    states = rn(B, W, 15, scale=0.5)
    states[..., -1] = (torch.rand(B, W, generator=g) < 0.5).float() * 2 - 1
    actions = torch.rand(B, W, 7, generator=g) * 2 - 1
    actions[..., 6] = (torch.rand(B, W, generator=g) < 0.5).float() * 2 - 1
    out = dict(images_primary=rn(B, W, 3, 224, 224).to(dtype), images_wrist=rn(B, W, 3, 224, 224).to(dtype),
               text=text.long(), states=states.to(dtype), actions=actions.to(dtype))
    if heads.get("depth"):
        out["depth_primary"] = (torch.rand(B, W, 1, 224, 224, generator=g) * 4.9 + 0.1).to(dtype)
        out["depth_wrist"] = (torch.rand(B, W, 1, 224, 224, generator=g) * 4.9 + 0.1).to(dtype)
    if heads.get("dino"):
        out["dino_primary"], out["dino_wrist"] = rn(B, W, 256, 768).to(dtype), rn(B, W, 256, 768).to(dtype)
    if heads.get("sam"):
        out["sam_primary"], out["sam_wrist"] = rn(B, W, 256, 256).to(dtype), rn(B, W, 256, 256).to(dtype)
    if heads.get("traj") or heads.get("flow_mask"):
        out["tracks"], out["tracks_gripper"] = rn(B, W, 784, 2, scale=2.0).to(dtype), rn(B, W, 784, 2, scale=2.0).to(dtype)
    if pin:
        return {k: v.pin_memory() for k, v in out.items()}
    return {k: v.to(device) for k, v in out.items()}


def batch_to_host_dict(batch_calvin):
    """The 13-tuple of the reference's collator (data_utils.py:1395-1397) -> the dict of HOST tensors used here
    (train_utils.py:99-123 picks the same entries)."""
    tr = batch_calvin[12] or {}
    out = dict(images_primary=batch_calvin[0], text=batch_calvin[1], actions=batch_calvin[2], images_wrist=batch_calvin[3],
               states=batch_calvin[4])
    for key, idx in (("depth_primary", 6), ("depth_wrist", 7), ("dino_primary", 8), ("dino_wrist", 9),
                     ("sam_primary", 10), ("sam_wrist", 11)):
        if batch_calvin[idx] is not None:
            out[key] = batch_calvin[idx]
    if "tracks" in tr:
        out["tracks"], out["tracks_gripper"] = tr["tracks"], tr["tracks_gripper"]
    return out


def batch_from_tuple(batch_calvin, device, dtype=torch.bfloat16):
    """13-tuple -> dict of device tensors (floating point entries cast to `dtype` ON THE DEVICE: a cross-device copy with a
    dtype change would convert on the host first)."""
    out = {}
    for k, v in batch_to_host_dict(batch_calvin).items():
        d = v.to(device, non_blocking=True)
        out[k] = d.to(dtype) if d.is_floating_point() else d
    return out


class _DeviceSlot:
    """One persistent set of device input buffers of the prefetcher (+ staging buffers for entries whose host dtype differs)."""

    def __init__(self):
        self.bufs, self.stage, self.consumed = {}, {}, None

    def fill(self, host, device, dtype):
        for k, v in host.items():
            want = dtype if v.is_floating_point() else v.dtype
            buf = self.bufs.get(k)
            if buf is None or buf.shape != v.shape or buf.dtype != want:
                buf = self.bufs[k] = torch.empty(v.shape, dtype=want, device=device)
            if v.dtype == want:
                buf.copy_(v, non_blocking=True)
            else:                                   # H2D in the host dtype, cast on the device
                st = self.stage.get(k)
                if st is None or st.shape != v.shape or st.dtype != v.dtype:
                    st = self.stage[k] = torch.empty(v.shape, dtype=v.dtype, device=device)
                st.copy_(v, non_blocking=True)
                buf.copy_(st)
        for k in [k for k in self.bufs if k not in host]:
            del self.bufs[k]
        return dict(self.bufs)


def prefetch_to_device(loader, device, to_host_dict=None, dtype=torch.bfloat16, slots=2):
    """Iterate `loader`, yielding each batch as a dict of DEVICE tensors; the host->device copies of batch i+1 are enqueued on a
    copy stream right after the consumer has enqueued step i, so a step's input transfer (193 MB at C2, ~3.5 ms over PCIe 5
    x16) runs beside that step's kernels.  The host stays at most one step ahead of the device (see `stage`).

    `to_host_dict(item)` maps a loader item to a dict of host tensors (default: the item itself); pinned host memory is
    needed for the copy to be asynchronous.  The device buffers are `slots` persistent sets reused round-robin (no allocator
    traffic, no cudaMalloc in steady state): a yielded dict stays valid until the consumer has asked for `slots - 1` more
    batches -- consume it (or copy it) before that, as the training loop and the CUDA-graph step's static-buffer copy do.
    Floating-point entries arrive as `dtype`.  On a CPU device this is a plain map (host logic is testable without a GPU)."""
    device = torch.device(device) if not isinstance(device, torch.device) else device
    to_host_dict = to_host_dict or (lambda item: item)
    if device.type != "cuda":
        for item in loader:
            yield {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in to_host_dict(item).items()}
        return
    copy_stream = torch.cuda.Stream(device)
    it = iter(loader)
    ring = [_DeviceSlot() for _ in range(max(2, slots))]

    def stage(i):
        try:
            item = next(it)
        except StopIteration:
            return None
        slot = ring[i % len(ring)]
        if slot.consumed is not None:
            # HOST-side wait for the step that read this slot's buffers (it finished long ago unless the host runs more than a
            # step ahead).  A device-side wait (copy_stream.wait_event) would park the copy in the stream's hardware queue
            # until the event fires; with the overlapped NCCL all-reduces of the data-parallel step in flight, copies parked
            # or released at arbitrary points of the step delay the step by an unpredictable amount
            slot.consumed.synchronize()
        with torch.cuda.stream(copy_stream):
            dev = slot.fill(to_host_dict(item), device, dtype)
            ready = torch.cuda.Event()
            ready.record(copy_stream)
        return dev, ready, slot

    i = 0
    nxt = stage(i)
    while nxt is not None:
        dev, ready, slot = nxt
        cur = torch.cuda.current_stream(device)
        cur.wait_event(ready)
        yield dev                                          # the consumer enqueues step i on `cur`
        cur = torch.cuda.current_stream(device)
        slot.consumed = torch.cuda.Event(blocking=True)    # blocking: the host thread sleeps in synchronize() instead of spinning
        slot.consumed.record(cur)
        i += 1
        nxt = stage(i)                                     # batch i+1 moves while step i runs


def train_one_epoch_calvin(args, model, epoch, calvin_loader, optimizer, lr_scheduler, device_id, wandb):
    """Drop-in for reference train_utils.py:59-68.  `model` is the bare DreamVLA or an object with `.module`; `optimizer`
    may be None (the fused flat AdamW of this package is used) -- `lr_scheduler`, when given, only supplies the lr."""
    core = model.module if hasattr(model, "module") else model
    core.train()
    state = getattr(core, "_dvla_train_step", None)
    if state is None:
        import torch.distributed as dist
        world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        state = TrainStep(core, StepConfig.from_args(args), world_size=world)
        core._dvla_train_step = state
    step_time_m, data_time_m = AverageMeter(), AverageMeter()
    end = time.time()
    dev = torch.device("cuda", device_id) if isinstance(device_id, int) else torch.device(device_id)
    # --cuda_graph: after ONE eager step (allocator pools, NCCL communicator and lazy tables are warm) the micro-step and the
    # optimiser step are captured once and replayed for every later batch of the same shapes (gradient accumulation 1 only)
    use_graph = bool(getattr(args, "cuda_graph", False)) and (args.gradient_accumulation_steps == 1
                                                               or state.cfg.reduce_every_micro_step)
    n_batches = getattr(calvin_loader, "num_batches", None)
    accum = args.gradient_accumulation_steps
    state.micro = 0           # the reference counts accumulation windows from the start of each epoch (:602)
    graphed = getattr(core, "_dvla_graphed_step", None)
    device_augment = bool(getattr(args, "device_augment", False)) and (getattr(args, "rgb_pad", -1) != -1
                                                                        or getattr(args, "gripper_pad", -1) != -1)
    for num_steps, batch in enumerate(prefetch_to_device(calvin_loader, dev, batch_to_host_dict)):
        data_time_m.update(time.time() - end)
        if device_augment:        # the collator's random shifts (reference data_utils.py:1337-1354), on the device
            from .data_utils import augment_batch
            batch = augment_batch(batch, args.rgb_pad, args.gripper_pad, bool(getattr(args, "traj_cons", False)))
        lr = lr_scheduler.get_last_lr()[0] if lr_scheduler is not None else args.learning_rate
        if use_graph and graphed is None and state.total_micro > 0:
            graphed = GraphedTrainStep(state, batch, warmup=0)
            core._dvla_graphed_step = graphed
        replay = graphed is not None and batch.keys() == graphed.static.keys() and \
            all(batch[k].shape == graphed.static[k].shape for k in batch)
        # optimiser step on accumulation boundaries AND on the last batch of the epoch (train_utils.py:602-604)
        boundary = (num_steps + 1) % accum == 0 or (n_batches is not None and num_steps == n_batches - 1)
        loss = graphed(batch, lr=lr, boundary=boundary) if replay else state(batch, lr=lr, boundary=boundary)
        if boundary:
            if lr_scheduler is not None:
                lr_scheduler.step()
            step_time_m.update(time.time() - end)
            end = time.time()
            if getattr(args, "rank", 0) == 0 and wandb is not None and getattr(args, "report_to_wandb", False):
                sps = args.gradient_accumulation_steps * args.batch_size * state.world_size / step_time_m.val
                wandb.log({"calvin_samples_per_second": sps, "loss_calvin": float(loss)}, commit=True)
    return state
