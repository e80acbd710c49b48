"""DreamVLA on sm_90a kernels -- drop-in mirror of reference models/dreamvla_model.py:122-991.

Same constructor kwargs, `forward(image_primary, image_wrist, state, text_token, action=None, track_infos=None,
action_label=None, mode='train')` -> the same 10-tuple, same parameter names / shapes (state_dict-compatible, incl. HF
Conv1D [in,out] weights), same attributes read by the entry points (`image_processor`, `clip_model`, `vision_encoder`,
`perceiver_resampler`, `transformer_backbone`, `*_decoder`, `action_model`, `_init_model_type()`, `sequence_length`).

What differs, by design (H100-first, results identical up to bf16 rounding):
  * every Linear/LayerNorm/attention runs on libdvla_sm90.so (wgmma GEMM with fused bias/act/residual/dropout
    epilogues, flash attention with the reference's {0,-inf} mask as a bit matrix + tile skipping);
  * both cameras go through the ViT / resampler in ONE batched call (the reference makes two, :672-673,:716-717);
  * the ViT patch-token permutation of random_masking(…, 0.0) is skipped (outputs invariant, see vit_mae.py here);
  * identical sentences are CLIP-encoded once.
Out of scope (need code/weights that are not in the reference tree, SURVEY §8a): use_dinosiglip, use_gpt2_pretrained,
use_dpt_head.  They raise NotImplementedError.
"""
from __future__ import annotations

import os
from functools import partial

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from .. import ops
from . import clip_text
from .action_model import ActionModel, ActionModelFM
from .gpt2 import GPT2Config, GPT2Model
from .layers import Block, LayerNorm, Linear
from .perceiver_resampler import PerceiverResampler
from .vit_mae import MaskedAutoencoderViT, get_1d_sincos_pos_embed_from_grid, get_2d_sincos_pos_embed  # noqa: F401


def generate_attention_mask(K, num_A, num_B, atten_goal, atten_goal_state, atten_only_obs, attn_robot_proprio_state,
                            mask_l_obs_ratio, num_obs_token, action_pred_steps):
    """Additive {0,-inf} mask [L, L], L = (num_A + num_B) * K.  Same rules, order of application and np.random call
    sequence as reference dreamvla_model.py:25-66 (bit-exact, tests/test_mask_cpu.py)."""
    n = num_A + num_B
    L = n * K
    mask = torch.zeros((L, L))
    ninf = -float("inf")
    for i in range(K):
        s = i * n
        e = s + n
        mask[s:e, e:] = ninf                      # no attention to later timesteps (:41)
        mask[:, s + num_A:e] = ninf               # B tokens are never attended to (:44)
        a0 = s + num_A + num_obs_token            # first action row of this timestep
        a1 = a0 + action_pred_steps
        if num_obs_token > 0 and action_pred_steps:
            mask[a0:a1, s + num_A:s + num_A + num_obs_token] = 0.0     # action rows see own obs/query cols (:48)
        if num_obs_token > 0 and atten_only_obs and action_pred_steps:
            mask[a0:a1] = ninf                                          # (:50)
            mask[a0:a1, s + 2:s + num_A] = 0.0                          # image tokens of the own step (:51)
            mask[a0:a1, s + num_A:s + num_A + num_obs_token] = 0.0      # (:52)
            if attn_robot_proprio_state:
                mask[a0:a1, s + 1:s + 2] = 0.0                          # (:54)
            if mask_l_obs_ratio > 0:
                count = int(mask_l_obs_ratio * num_obs_token)
                selected = np.random.choice(range(num_obs_token), size=count, replace=False)
                for num in selected:
                    mask[a0:a1, s + num_A + num] = ninf                 # (:59)
        if num_obs_token > 0 and atten_goal:
            if i < K - atten_goal:
                pe = (i + atten_goal) * n
                if atten_goal_state:
                    mask[s + num_A:s + num_A + num_obs_token, pe + 1:pe + 2] = 0.0   # (:64)
    return mask


def prune_closure(vis, sel, n_tok):
    """Token indices (ascending) a rollout keeps for timestep `sel` under the visibility matrix vis [L, L] (bool): every slot
    of timestep sel plus, transitively, every slot a kept row can see."""
    keep = torch.zeros(vis.shape[0], dtype=torch.bool)
    keep[sel * n_tok:(sel + 1) * n_tok] = True               # every slot of the selected timestep
    while True:                                              # + everything a kept row can see (transitively)
        grown = keep | vis[keep].any(dim=0)
        if bool((grown == keep).all()):
            return keep.nonzero().flatten()
        keep = grown


def batched_rollout_layout(vis, S, n_a, action_pred_steps):
    """Per timestep sel of a window of S: idx_sel = prune_closure(sel) + the A slots (the first n_a of a timestep) of the
    timesteps after sel, in token order, and the position of sel's first action row in it.  Every idx_sel must have the same
    length and start with the pruned single-env sequence (then a batch of envs at any mix of sel shares one sequence length,
    and each env's kept rows compute what they compute alone); ValueError otherwise.  -> (idx [S, Lb] int64, r0 [S] int64)."""
    n_tok = vis.shape[0] // S
    rows, r0s = [], []
    for sel in range(S):
        kept = prune_closure(vis, sel, n_tok)
        want = torch.zeros(vis.shape[0], dtype=torch.bool)
        want[kept] = True
        for t in range(sel + 1, S):
            want[t * n_tok:t * n_tok + n_a] = True
        idx = want.nonzero().flatten()
        if not torch.equal(idx[:len(kept)], kept):
            raise ValueError(f"batched rollout: under this attention mask the pruned sequence of timestep {sel} is not a prefix "
                             "of its batched layout; use rollout_action per env")
        rows.append(idx)
        a0 = sel * n_tok + n_tok - action_pred_steps            # first action row of timestep sel
        r0s.append(int((kept < a0).sum()))
    lens = sorted({len(r) for r in rows})
    if len(lens) != 1:
        raise ValueError(f"batched rollout: the kept-token count differs between timesteps ({lens}) under this attention "
                         "mask, so the envs cannot share one batch; use rollout_action per env")
    return torch.stack(rows), torch.tensor(r0s, dtype=torch.long)


class _WorldDecoder(nn.Module):
    """Helper that RUNS one world-knowledge decoder (reference :793-911); it owns no parameters -- the parameters stay
    on DreamVLA under the reference names.

    Reference computation per sequence: x = cat(projector(queries) [n_per], mask_token x n_mask) + pos_emb -> 2 timm Blocks
    -> LayerNorm -> Linear on the n_mask rows.  95 % of the rows are mask tokens, and `mask_token + pos_emb[n_per:]` does not
    depend on the sequence (SURVEY §8 f-4), which is used twice:
      * shared first block input: LayerNorm-1 and the QKV projection of the mask rows of block 0 are computed ONCE per call
        ([n_mask, D] rows instead of n_seq * n_mask); the per-sequence rows are the n_per query rows only;
      * identical mask rows: if all mask rows of pos_emb are equal (the SAM head: zero position embedding, reference
        :414-415 / :558-564), the n_mask mask tokens of a sequence are the same vector at every depth (every layer is
        row-wise or a softmax over the same keys), so the decoder runs on n_per + 1 rows and the attention sees the shared
        row's key / value n_mask times; the prediction of that row is every mask row's prediction.
    Both are identities in exact arithmetic; in bf16 only summation orders change."""

    _identical_cache = {}

    @staticmethod
    def _mask_rows_identical(pos_emb, n_per):
        key = (pos_emb.data_ptr(), pos_emb._version, n_per)
        c = _WorldDecoder._identical_cache
        if key not in c:
            if len(c) > 64:
                c.clear()
            rows = pos_emb.detach()[0, n_per:]
            c[key] = bool((rows == rows[:1]).all().item())        # one host read per parameter version (before any capture)
        return c[key]

    _bias_cache = {}

    @staticmethod
    def _repeat_bias(L, n_rep, device):
        """fp32 [L]: 0 for the distinct rows, log(n_rep) for the last one -- its key counts n_rep times in every softmax."""
        key = (L, n_rep, str(device))
        c = _WorldDecoder._bias_cache
        if key not in c:
            b = torch.zeros(L, dtype=torch.float32)
            b[-1] = float(np.log(n_rep))
            c[key] = b.to(device)
        return c[key]

    @staticmethod
    def _block_with_repeated_key(blk, x, n_per, n_rep):
        """timm Block on x [n, n_per + 1, D] whose last row stands for n_rep identical tokens: the n_per + 1 distinct rows are
        the queries and the keys; the shared row's score gets + log(n_rep), which is exactly softmax over n_rep copies of it."""
        n, L, D = x.shape
        at = blk.attn
        res, h = blk.norm1.fork(x)
        qkv = at.qkv(h).view(n, L, 3, at.num_heads, at.head_dim)
        o = ops.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], at.scale, key_bias=_WorldDecoder._repeat_bias(L, n_rep, x.device))
        x = at.proj(o.view(n, L, D), residual=res)
        res, h = blk.norm2.fork(x)
        return blk.mlp(h, residual=res)

    @staticmethod
    def run(feature, projector, mask_token, pos_emb, blocks, norm, pred, n_groups, n_per, n_mask, hidden, act=None):
        # feature [B, S, n_tok, D] -> projector -> [B*S*n_groups, n_per, hidden]
        B, S = feature.shape[:2]
        n = B * S * n_groups
        emb = projector(feature.reshape(-1, feature.shape[-1])).view(n, n_per, hidden)
        emb = emb + pos_emb[:, :n_per]
        if _WorldDecoder._mask_rows_identical(pos_emb, n_per):
            m = (mask_token + pos_emb[:, n_per:n_per + 1]).expand(n, 1, hidden)
            x = torch.cat((emb, m), dim=1)                                   # [n, n_per + 1, D]
            for blk in blocks:
                x = _WorldDecoder._block_with_repeated_key(blk, x, n_per, n_mask)
            y = pred(norm(x[:, n_per, :].contiguous()), act=act)             # [n, C]: every mask row's prediction
            return y.unsqueeze(1).expand(n, n_mask, -1)
        # block 0 with the mask rows' LayerNorm-1 + QKV shared across sequences
        blk = blocks[0]
        at = blk.attn
        m = (mask_token + pos_emb[:, n_per:])[0]                             # [n_mask, D], sequence independent
        qkv_e = at.qkv(blk.norm1(emb))                                       # [n, n_per, 3D]
        qkv_m = at.qkv(blk.norm1(m))                                         # [n_mask, 3D]   (once)
        qkv = ops.cat_broadcast(qkv_e, qkv_m).view(n, n_per + n_mask, 3, at.num_heads, at.head_dim)
        o = ops.self_attention_fused(qkv, at.scale)
        x = ops.cat_broadcast(emb, m)                                        # the block's input (residual branch)
        x = at.proj(o.view(n, n_per + n_mask, hidden), residual=x)
        res, h = blk.norm2.fork(x)
        x = blk.mlp(h, residual=res)
        for blk in list(blocks)[1:]:
            x = blk(x)
        x = norm(x[:, -n_mask:, :].reshape(-1, hidden))
        return pred(x, act=act)


class DreamVLA(nn.Module):
    def __init__(
        self,
        finetune_type,
        clip_device,
        vit_checkpoint_path,
        sequence_length=10,
        num_resampler_query=9,
        num_obs_token_per_image=10,
        obs_pred=False,
        atten_only_obs=False,
        attn_robot_proprio_state=False,
        atten_goal=False,
        atten_goal_state=False,
        mask_l_obs_ratio=0.0,
        calvin_input_image_size=224,
        patch_size=16,
        mask_ratio=0.0,
        num_token_per_timestep=41,
        input_self=False,
        action_pred_steps=1,
        transformer_layers=12,
        hidden_dim=384,
        transformer_heads=12,
        phase="",
        gripper_width=False,
        pred_num=1,
        depth_pred=False,
        trajectory_pred=False,
        use_depth_query=False,
        use_dpt_head=False,
        use_trajectory_query=False,
        track_label_patch_size=4,
        dino_feat_pred=False,
        sam_feat_pred=False,
        use_dinosiglip=False,
        use_dit_head=False,
        use_gpt2_pretrained=False,
        no_pred_gripper_traj=False,
        no_unshuffle=False,
        share_query=False,
        attn_implementation=False,
        use_fm=False,
        dit_type="DiT-B",
    ):
        super().__init__()
        for flag, name in ((use_dinosiglip, "use_dinosiglip"), (use_gpt2_pretrained, "use_gpt2_pretrained"),
                           (use_dpt_head, "use_dpt_head")):
            if flag:
                raise NotImplementedError(f"{name}: needs weights/code outside the reference tree (out of scope, SURVEY §8a)")
        self.finetune_type = finetune_type
        self.device = clip_device
        self.sequence_length = sequence_length
        self.action_pred_steps = action_pred_steps
        self.obs_pred = obs_pred
        self.depth_pred = depth_pred
        self.dino_feat_pred = dino_feat_pred
        self.sam_feat_pred = sam_feat_pred
        self.trajectory_pred = trajectory_pred
        self.atten_goal = atten_goal
        self.atten_goal_state = atten_goal_state
        self.atten_only_obs = atten_only_obs
        self.attn_robot_proprio_state = attn_robot_proprio_state
        self.mask_l_obs_ratio = mask_l_obs_ratio
        self.hidden_dim = hidden_dim
        self.phase = phase
        self.dit_type = dit_type
        assert self.phase in ["pretrain", "finetune", "evaluate"]
        self.share_query = share_query
        self.gripper_width = gripper_width
        self.vit_checkpoint_path = vit_checkpoint_path
        self.pred_num = pred_num
        self.use_dinosiglip = False
        D = hidden_dim

        self.text_projector = Linear(512, D)
        self.arm_state_encoder = Linear(6, D)
        self.gripper_state_encoder = Linear(2, D)
        self.state_projector = Linear(2 * D, D)
        # action encoders exist in the reference (:203-205) but are never used in forward
        self.action_pose_encoder = Linear(6, D)
        self.action_gripper_position_encoder = Linear(2, D)
        self.action_projector = Linear(2 * D, D)

        self.vision_encoder = MaskedAutoencoderViT(patch_size=16, embed_dim=768, depth=12, num_heads=12,
                                                   decoder_embed_dim=512, decoder_depth=8, decoder_num_heads=16,
                                                   mlp_ratio=4, norm_layer=partial(LayerNorm, eps=1e-6))
        self.RESAMPLER_hidden_dim = 768
        self.NUM_RESAMPLER_QUERY = num_resampler_query
        self.perceiver_resampler = PerceiverResampler(dim=768, num_latents=num_resampler_query, depth=3)
        self.image_primary_projector = Linear(768, D)
        self.cls_token_primary_projector = Linear(768, D)
        self.image_wrist_projector = Linear(768, D)
        self.cls_token_wrist_projector = Linear(768, D)

        if self.action_pred_steps > 0:
            self.action_pred_token = nn.Parameter(torch.zeros(1, 1, self.action_pred_steps, D))

        self.NUM_OBS_TOKEN = self.NUM_DEPTH_TOKEN = self.NUM_TRAJ_TOKEN = self.NUM_DINO_TOKEN = self.NUM_SAM_TOKEN = 0
        if self.obs_pred:
            self.NUM_OBS_TOKEN_PER_IMAGE = num_obs_token_per_image
            self.NUM_OBS_TOKEN = num_obs_token_per_image * 2
            self.obs_tokens = nn.Parameter(torch.zeros(1, 1, self.NUM_OBS_TOKEN, D))
        if self.depth_pred:
            self.NUM_OBS_TOKEN_PER_DEPTH = num_obs_token_per_image
            self.NUM_DEPTH_TOKEN = num_obs_token_per_image * 2
        if self.dino_feat_pred:
            self.NUM_OBS_TOKEN_PER_DINO = num_obs_token_per_image
            self.NUM_DINO_TOKEN = num_obs_token_per_image * 2
        if self.sam_feat_pred:
            self.NUM_OBS_TOKEN_PER_SAM = num_obs_token_per_image
            self.NUM_SAM_TOKEN = num_obs_token_per_image * 2
        if self.trajectory_pred:
            self.NUM_OBS_TOKEN_PER_TRAJ = num_obs_token_per_image
            self.NUM_TRAJ_TOKEN = num_obs_token_per_image * (1 if no_pred_gripper_traj else 2)
        if not self.share_query:
            if self.depth_pred:
                self.depth_tokens = nn.Parameter(torch.zeros(1, 1, self.NUM_DEPTH_TOKEN, D))
            if self.dino_feat_pred:
                self.dino_feat_tokens = nn.Parameter(torch.zeros(1, 1, self.NUM_DINO_TOKEN, D))
            if self.sam_feat_pred:
                self.sam_feat_tokens = nn.Parameter(torch.zeros(1, 1, self.NUM_SAM_TOKEN, D))
            if trajectory_pred:
                self.trajectory_tokens = nn.Parameter(torch.zeros(1, 1, self.NUM_TRAJ_TOKEN, D))

        self.embedding_layer_norm = LayerNorm(D)
        self.attention_mask = nn.Parameter(self._make_mask(), requires_grad=False)
        self._mask_cache = None
        self._obs_drop_seed = self._obs_drop_mask = None      # see obs_drop_on_device
        self.transformer_backbone_position_embedding = nn.Parameter(torch.zeros(1, sequence_length, 1, D), requires_grad=True)
        config = GPT2Config()
        config.hidden_size = D
        config.n_layer = transformer_layers
        config.vocab_size = 1
        config.n_head = transformer_heads
        self.attn_implementation = config.attn_implementation = attn_implementation
        self.transformer_backbone = GPT2Model(config)

        MLP_hidden_dim = D // 2
        # unused in forward, kept for state_dict compatibility (:320-333)
        self.recon_state_decoder = nn.Sequential(Linear(D, MLP_hidden_dim), nn.ReLU(), Linear(MLP_hidden_dim, MLP_hidden_dim), nn.ReLU())
        self.recon_arm_state_decoder = nn.Sequential(Linear(MLP_hidden_dim, 6), nn.Tanh())
        self.recon_gripper_state_decoder = nn.Sequential(Linear(MLP_hidden_dim, 1), nn.Sigmoid())

        n_patch = int(calvin_input_image_size ** 2 / patch_size / patch_size) * pred_num
        q_in = int(D / 4) if share_query else D

        def two_blocks():
            return nn.Sequential(Block(D, num_heads=16, mlp_ratio=4, qkv_bias=True, eps=1e-5),
                                 Block(D, num_heads=16, mlp_ratio=4, qkv_bias=True, eps=1e-5))

        if self.obs_pred:
            self.IMAGE_DECODER_hidden_dim = D
            self.NUM_MASK_TOKEN = n_patch
            self.PATCH_SIZE = patch_size
            self.mask_token = nn.Parameter(torch.zeros(1, 1, D))
            self.image_decoder_obs_pred_projector = Linear(q_in, D)
            self.image_decoder_position_embedding = nn.Parameter(torch.zeros(1, num_obs_token_per_image + n_patch, D), requires_grad=False)
            self.image_decoder = two_blocks()
            self.image_decoder_norm = LayerNorm(D)
            self.image_decoder_pred = Linear(D, patch_size ** 2 * 3)
        if self.depth_pred:
            self.use_dpt_head = False
            self.DEPTH_DECODER_hidden_dim = D
            self.NUM_DEPTH_MASK_TOKEN = n_patch
            self.PATCH_SIZE = patch_size
            self.depth_decoder_obs_pred_projector = Linear(q_in, D)
            self.depth_decoder = two_blocks()
            self.depth_decoder_norm = LayerNorm(D)
            self.depth_decoder_pred = Linear(D, patch_size ** 2)
            self.depth_mask_token = nn.Parameter(torch.zeros(1, 1, D))
            self.depth_decoder_position_embedding = nn.Parameter(torch.zeros(1, num_obs_token_per_image + n_patch, D), requires_grad=False)
        if self.dino_feat_pred:
            self.DINO_DECODER_hidden_dim = D
            self.NUM_DINO_MASK_TOKEN = 256 * pred_num
            self.dino_decoder_obs_pred_projector = Linear(q_in, D)
            self.dino_feat_decoder = two_blocks()
            self.dino_decoder_norm = LayerNorm(D)
            self.dino_decoder_pred = Linear(D, 768)
            self.dino_mask_token = nn.Parameter(torch.zeros(1, 1, D))
            self.dino_decoder_position_embedding = nn.Parameter(torch.zeros(1, num_obs_token_per_image + 256 * pred_num, D), requires_grad=False)
        if self.sam_feat_pred:
            self.SAM_DECODER_hidden_dim = D
            self.NUM_SAM_MASK_TOKEN = 256 * pred_num
            self.sam_decoder_obs_pred_projector = Linear(q_in, D)
            self.sam_feat_decoder = two_blocks()
            self.sam_decoder_norm = LayerNorm(D)
            self.sam_decoder_pred = Linear(D, 256)
            self.sam_mask_token = nn.Parameter(torch.zeros(1, 1, D))
            self.sam_decoder_position_embedding = nn.Parameter(torch.zeros(1, num_obs_token_per_image + 256 * pred_num, D), requires_grad=False)
        if self.trajectory_pred:
            self.use_traj_query = use_trajectory_query
            self.track_label_patch_size = track_label_patch_size
            self.TRAJ_DECODER_hidden_dim = D
            if no_unshuffle:
                self.NUM_TRAJ_MASK_TOKEN = 784 * pred_num
                self.traj_decoder_pred = Linear(D, 2)
            else:
                self.NUM_TRAJ_MASK_TOKEN = n_patch
                self.traj_decoder_pred = Linear(D, (patch_size // track_label_patch_size) ** 2 * 2)
            self.PATCH_SIZE = patch_size
            self.traj_decoder_obs_pred_projector = Linear(D, D)
            self.traj_decoder = two_blocks()
            self.traj_decoder_norm = LayerNorm(D)
            self.traj_mask_token = nn.Parameter(torch.zeros(1, 1, D))
            torch.nn.init.normal_(self.traj_mask_token, std=0.02)
            self.traj_decoder_position_embedding = nn.Parameter(torch.zeros(1, num_obs_token_per_image + self.NUM_TRAJ_MASK_TOKEN, D), requires_grad=False)

        self.use_dit_head = use_dit_head
        self.use_fm = bool(use_fm) and bool(use_dit_head)
        if self.use_dit_head:
            action_model_cls = ActionModelFM if use_fm else ActionModel                   # :450
            self.action_model = action_model_cls(model_type=dit_type, token_size=D, in_channels=7,
                                                 future_action_window_size=self.action_pred_steps - 1, past_action_window_size=0)
        else:
            self.action_decoder = nn.Sequential(Linear(D, MLP_hidden_dim), nn.ReLU(), Linear(MLP_hidden_dim, MLP_hidden_dim), nn.ReLU())
            self.arm_action_decoder = nn.Sequential(Linear(MLP_hidden_dim, 6), nn.Tanh())
            self.gripper_action_decoder = nn.Sequential(Linear(MLP_hidden_dim, 1), nn.Sigmoid())
        self.initialize_weights()

        if vit_checkpoint_path is not None and os.path.exists(str(vit_checkpoint_path)):
            vit_checkpoint = torch.load(vit_checkpoint_path, map_location="cpu")
            self.vision_encoder.load_state_dict(vit_checkpoint["model"], strict=False)
        ckpt = "checkpoints/clip/ViT-B-32.pt"
        self.clip_model, self.image_processor = clip_text.load(ckpt if os.path.exists(ckpt) else "ViT-B/32", device=clip_device)

    # ------------------------------------------------------------------------------------------------------------------
    def _this_num_obs_token(self):
        if self.share_query:
            return self.NUM_OBS_TOKEN
        if self.obs_pred or self.depth_pred or self.trajectory_pred or self.dino_feat_pred or self.sam_feat_pred:
            return self.NUM_OBS_TOKEN + self.NUM_DEPTH_TOKEN + self.NUM_TRAJ_TOKEN + self.NUM_DINO_TOKEN + self.NUM_SAM_TOKEN
        return 0

    def _make_mask(self, mask_l_obs_ratio=None):
        n_obs = self._this_num_obs_token()
        ratio = self.mask_l_obs_ratio if mask_l_obs_ratio is None else mask_l_obs_ratio
        return generate_attention_mask(K=self.sequence_length, num_A=1 + 1 + self.NUM_RESAMPLER_QUERY * 2 + 1 * 2,
                                       num_B=n_obs + self.action_pred_steps, atten_goal=self.atten_goal,
                                       atten_goal_state=self.atten_goal_state, atten_only_obs=self.atten_only_obs,
                                       attn_robot_proprio_state=self.attn_robot_proprio_state,
                                       mask_l_obs_ratio=ratio, num_obs_token=n_obs,
                                       action_pred_steps=self.action_pred_steps)

    @property
    def redraws_mask(self):
        """True when every training forward draws a fresh observation-token drop (reference :610-628 with :55-59)."""
        return self.phase == "pretrain" and self.mask_l_obs_ratio > 0 and self.atten_only_obs

    @property
    def obs_drop_on_device(self):
        """Whether a training forward that redraws the mask (`redraws_mask`) draws it on the device (ops.ObsDropMask, one
        kernel, capturable in a CUDA graph) instead of through np.random on the host (the reference's call sequence, a
        host-device round trip per forward).  Switching it on fixes the draw's seed from torch's default generator."""
        return self._obs_drop_seed is not None

    @obs_drop_on_device.setter
    def obs_drop_on_device(self, on):
        if not on:
            self._obs_drop_seed = self._obs_drop_mask = None
        elif not self.obs_drop_on_device:
            self._obs_drop_seed = int(torch.randint(0, 2 ** 63 - 1, (1,)))
            self._obs_drop_mask = None
            if self.attention_mask.is_cuda:     # allocate now: the first draw may be inside a CUDA-graph capture
                self._device_obs_drop(self.attention_mask.device)

    def _device_obs_drop(self, device):
        """The model's ops.ObsDropMask on `device`, built from the mask without the drop (mask_l_obs_ratio = 0)."""
        m = self._obs_drop_mask
        if m is None or m.bits.device != torch.device(device):
            n_obs = self._this_num_obs_token()
            m = self._obs_drop_mask = ops.ObsDropMask(
                self._make_mask(mask_l_obs_ratio=0.0) == 0, device, K=self.sequence_length,
                num_A=1 + 1 + self.NUM_RESAMPLER_QUERY * 2 + 1 * 2, n_obs=n_obs, n_act=self.action_pred_steps,
                count=int(self.mask_l_obs_ratio * n_obs), seed=self._obs_drop_seed)      # count as the reference's (:57)
        return m

    def _attn_mask(self, device):
        """Bit-matrix form of self.attention_mask, rebuilt when the parameter changes (pretrain phase / load_state_dict)."""
        key = (self.attention_mask.data_ptr(), self.attention_mask._version, str(device))
        if self._mask_cache is None or self._mask_cache[0] != key:
            self._mask_cache = (key, ops.AttnMask.from_additive(self.attention_mask.detach().float().cpu(), device))
        return self._mask_cache[1]

    def initialize_weights(self):  # reference :543-579
        def sincos(dim, n_obs, n_mask):
            a = get_2d_sincos_pos_embed(dim, int(n_obs ** 0.5), cls_token=False)
            b = get_2d_sincos_pos_embed(dim, int(n_mask ** 0.5), cls_token=False)
            return torch.from_numpy(np.concatenate((a, b), axis=0)).float().unsqueeze(0)
        if self.obs_pred:
            self.image_decoder_position_embedding.data.copy_(sincos(self.hidden_dim, self.NUM_OBS_TOKEN_PER_IMAGE, self.NUM_MASK_TOKEN))
            torch.nn.init.normal_(self.mask_token, std=0.02)
        if self.depth_pred:
            self.depth_decoder_position_embedding.data.copy_(sincos(self.hidden_dim, self.NUM_OBS_TOKEN_PER_DEPTH, self.NUM_DEPTH_MASK_TOKEN))
            torch.nn.init.normal_(self.depth_mask_token, std=0.02)
        # sam: position embedding stays zero and the mask token zero-initialised (reference :558-564 is commented out)
        if self.dino_feat_pred:
            self.dino_decoder_position_embedding.data.copy_(sincos(self.hidden_dim, self.NUM_OBS_TOKEN_PER_DINO, self.NUM_DINO_MASK_TOKEN))
            torch.nn.init.normal_(self.dino_mask_token, std=0.02)
        if self.trajectory_pred:
            self.traj_decoder_position_embedding.data.copy_(sincos(self.hidden_dim, self.NUM_OBS_TOKEN_PER_TRAJ, self.NUM_TRAJ_MASK_TOKEN))
            torch.nn.init.normal_(self.traj_mask_token, std=0.02)
        torch.nn.init.normal_(self.transformer_backbone_position_embedding, std=0.02)
        self.apply(self._init_weights)

    def _init_weights(self, m):  # reference :581-591 (Conv1D is not nn.Linear: GPT-2 keeps its own init)
        if isinstance(m, nn.Linear):
            torch.nn.init.xavier_uniform_(m.weight)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            if m.weight is not None:
                nn.init.constant_(m.weight, 1.0)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)

    def _init_model_type(self):  # reference :593-603
        self.vision_encoder_type = next(self.vision_encoder.parameters()).type()
        self.perceiver_resampler_type = next(self.perceiver_resampler.parameters()).type()
        self.transformer_backbone_type = next(self.transformer_backbone.parameters()).type()
        if not self.use_dit_head:
            self.action_decoder_type = next(self.action_decoder.parameters()).type()

    # ------------------------------------------------------------------------------------------------------------------
    def _encode_state(self, st):
        """reference :656-664.  st [n, 7] (arm 6 + open/closed flag) or [n, 8] (--gripper_width) -> [n, D]."""
        dt = torch.bfloat16
        st = st.to(dt)
        arm_state_feature = self.arm_state_encoder(st[:, :6].contiguous())
        if not self.gripper_width:
            idx = (st[:, 6:].flatten() >= 1).long()      # 0 if < 1 else 1 (no host scalars: graph-capturable)
            idxf = idx.to(dt)
            gripper_in = torch.stack((1 - idxf, idxf), dim=1)      # == F.one_hot(idx, 2), without its value check
        else:
            gripper_in = st[:, 6:].contiguous()
        gripper_state_feature = self.gripper_state_encoder(gripper_in)
        return self.state_projector(torch.cat((arm_state_feature, gripper_state_feature), dim=1))

    def _encode_vision(self, image_primary, image_wrist):
        """reference :666-673, :716-737 for n frames of both cameras in ONE ViT / resampler batch.
        [n, 3, 224, 224] x2 -> (primary tokens [n, nq, D], wrist tokens [n, nq, D], cls_primary [n, 1, D], cls_wrist [n, 1, D])."""
        dt = torch.bfloat16
        n = image_primary.shape[0]
        D = self.hidden_dim
        with torch.no_grad():
            imgs = torch.cat((image_primary, image_wrist), dim=0).to(dt)
            feats, _, _ = self.vision_encoder.forward_encoder(imgs, mask_ratio=0.0)        # [2n, 197, 768]
        cls_tok = feats[:, 0, :]                                                            # [2n, 768]
        patches = feats[:, 1:, :]                                                           # [2n, 196, 768]
        resampled = self.perceiver_resampler(patches.unsqueeze(1).unsqueeze(1))            # [2n, 1, nq, 768]
        resampled = resampled.reshape(2, n * self.NUM_RESAMPLER_QUERY, 768)
        pe = self.image_primary_projector(resampled[0]).view(n, -1, D)
        we = self.image_wrist_projector(resampled[1]).view(n, -1, D)
        cp = self.cls_token_primary_projector(cls_tok[:n].contiguous()).view(n, 1, D)
        cw = self.cls_token_wrist_projector(cls_tok[n:].contiguous()).view(n, 1, D)
        return pe, we, cp, cw

    def _query_tokens(self):
        """The learned B-slot tokens of one timestep, in slot order (:745-757): obs, depth, dino, sam, traj, action."""
        parts = []
        if self.obs_pred:
            parts.append(self.obs_tokens)
        if not self.share_query:
            if self.depth_pred:
                parts.append(self.depth_tokens)
            if self.dino_feat_pred:
                parts.append(self.dino_feat_tokens)
            if self.sam_feat_pred:
                parts.append(self.sam_feat_tokens)
            if self.trajectory_pred:
                parts.append(self.trajectory_tokens)
        if self.action_pred_steps > 0:
            parts.append(self.action_pred_token)
        return parts

    FUSED_SAMPLER = True

    def _fused_sampler_fits(self, bs):
        """One sequence (rollouts: 12 rows), 3 action steps, head_dim 64 or 96, no autograd: the whole guided sampler loop runs
        as one persistent kernel (csrc/dit_sampler.cu)."""
        net = self.action_model.net
        return (self.FUSED_SAMPLER and 4 * bs * self.action_pred_steps <= 12 and self.action_pred_steps == 3
                and net.x_embedder.linear.weight.shape[0] in (64 * net.num_heads, 96 * net.num_heads)
                and not torch.is_grad_enabled())

    def _ddim_actions(self, feat, sample_noise, dev):
        """10-step DDIM with classifier-free guidance 1.5 (:935-987) on feat [n, action_pred_steps, D] -> [n, steps, 7]."""
        bs = feat.shape[0]
        fused = self._fused_sampler_fits(bs)
        cfg_scale = 1.5
        if self.use_fm:
            # --use_fm (ActionModelFM / FMDiffusion, respace.py:118-191): the sampler forces the guidance scale to 1.0, ignores
            # the noise it is handed and draws its own start state [2 bs, steps, 7]; `sample_noise` (parity tests) injects
            # that state ([2 bs, ...], or [bs, ...] used for both halves -- only the first half reaches the output)
            if self.action_model.ddim_diffusion is None:
                self.action_model.create_ddim(ddim_step=10)
            shape = (2 * bs, self.action_pred_steps, self.action_model.in_channels)
            if fused and self.action_model.ddim_diffusion.num_timesteps <= 12:
                # the same start-state draw as FMDiffusion (the CUDA generator advances alike on both paths); the kernel
                # integrates the first half, the only one that reaches the output
                start = sample_noise if sample_noise is not None else torch.randn(*shape, device=dev)
                from .. import _lib as L
                return L.dit_fm_sample(self.action_model.net, self.action_model.ddim_diffusion, feat.to(torch.bfloat16),
                                       start[:bs].to(device=dev, dtype=torch.float32)).to(feat.dtype)
            uncondition = self.action_model.net.z_embedder.uncondition.unsqueeze(0).expand(bs, self.action_pred_steps, -1)
            z = torch.cat([feat, uncondition], 0)
            start = None
            if sample_noise is not None:
                start = sample_noise if sample_noise.shape[0] == 2 * bs else torch.cat([sample_noise, sample_noise], 0)
            samples = self.action_model.ddim_diffusion.ddim_sample_loop(
                self.action_model.net.forward_with_cfg, shape, None, clip_denoised=False,
                model_kwargs=dict(z=z, cfg_scale=cfg_scale), device=dev, eta=0.0, start=start)
            return samples.chunk(2, dim=0)[0].to(feat.dtype)
        if sample_noise is None:
            sample_noise = torch.randn(bs, self.action_pred_steps, self.action_model.in_channels, device=dev)
        noise = sample_noise.to(device=dev, dtype=feat.dtype)
        noise = torch.cat([noise, noise], 0)
        uncondition = self.action_model.net.z_embedder.uncondition.unsqueeze(0).expand(bs, self.action_pred_steps, -1)
        z = torch.cat([feat, uncondition], 0)
        if self.action_model.ddim_diffusion is None:
            self.action_model.create_ddim(ddim_step=10)
        net = self.action_model.net
        if fused:
            # rollouts: the whole guided DDIM loop as one persistent kernel (csrc/dit_sampler.cu)
            from .. import _lib as L
            return L.dit_ddim_sample(net, self.action_model.ddim_diffusion, feat.to(torch.bfloat16), noise[:bs].float(),
                                     cfg_scale).to(feat.dtype)
        samples = self.action_model.ddim_diffusion.ddim_sample_loop(
            self.action_model.net.forward_with_cfg, noise.shape, noise, clip_denoised=False,
            model_kwargs=dict(z=z, cfg_scale=cfg_scale), device=dev, eta=0.0)
        samples, _ = samples.chunk(2, dim=0)
        return samples

    # ---- rollout-level incremental inference (SURVEY §8 f-1; reference utils/eval_utils_calvin.py:82-147) --------------
    @torch.no_grad()
    def encode_text_embedding(self, text_token):
        """text_token int [n, 77] -> projected text slot [n, D] (:643-653).  Frozen for an episode by the rollout wrapper."""
        tf = self.clip_model.encode_text(text_token.contiguous()).to(torch.bfloat16)
        return self.text_projector(tf)

    @torch.no_grad()
    def encode_frame_tokens(self, image_primary, image_wrist, state):
        """Per-frame, position-independent slots of n frames: [state(1) . primary nq . wrist nq . cls_p . cls_w] -> [n, 35, D].
        A frame's block depends on that frame only (ViT, resampler and projectors never mix frames), so a rollout can keep
        it across env steps instead of re-encoding the whole window (the reference re-runs all S frames every step)."""
        st = self._encode_state(state).unsqueeze(1)
        pe, we, cp, cw = self._encode_vision(image_primary, image_wrist)
        return torch.cat((st, pe, we, cp, cw), dim=1)

    def _rollout_mask(self, sel, prune, device):
        """AttnMask of the tokens kept for selected timestep `sel`.  prune=False: the full [L, L] mask.  prune=True: the slots
        of timestep `sel` plus, transitively, every slot one of the kept rows can see -- for the finetune / evaluate masks
        that is the A slots of timesteps 0..sel and the B slots of `sel` (later timesteps are hidden by :41, B slots of other
        timesteps by :44).  A dropped token is visible to no kept row, so the kept rows' attention is unchanged."""
        if not prune:
            return self._attn_mask(device), None, None
        key = (self.attention_mask.data_ptr(), self.attention_mask._version, sel, str(device))
        cache = self.__dict__.setdefault("_rollout_mask_cache", {})
        if key not in cache:
            n_tok = self.attention_mask.shape[0] // self.sequence_length
            vis = (self.attention_mask.detach().float().cpu() == 0)
            idx = prune_closure(vis, sel, n_tok)
            cache[key] = (ops.AttnMask.from_additive(self.attention_mask.detach().float().cpu()[idx][:, idx].contiguous(),
                                                     device), idx.to(device), idx)
        return cache[key]

    def _batched_rollout_tables(self, device):
        """`batched_rollout_layout` of the model's mask, built on the host once per mask and device -> (AttnMaskStack of the S
        masks M[idx_sel][:, idx_sel], idx [S, Lb], first action row [S]) on the device.  For the finetune / evaluate masks
        idx_sel is A slots 0..sel, B slots of sel, A slots sel+1..S-1 (36*S + n_B tokens for every sel); no kept row sees the
        appended A slots (:41)."""
        key = (self.attention_mask.data_ptr(), self.attention_mask._version, str(device))
        cache = self.__dict__.setdefault("_batched_rollout_cache", {})
        if key not in cache:
            vis = self.attention_mask.detach().float().cpu() == 0
            idx, r0 = batched_rollout_layout(vis, self.sequence_length, 1 + 1 + 2 * self.NUM_RESAMPLER_QUERY + 2,
                                             self.action_pred_steps)
            stack = ops.AttnMaskStack(torch.stack([vis[r][:, r] for r in idx]), device)
            cache[key] = (stack, idx.to(device), r0.to(device))
        return cache[key]

    @torch.no_grad()
    def rollout_actions(self, text_embedding, frame_tokens, sel, sample_noise=None, return_features=False):
        """`rollout_action(..., sel[e], prune=True)` for N envs in one batch: one backbone pass over N sequences of equal length
        (`_batched_rollout_tables`), each under its own mask, then one sampler call for the N action-token groups.

        text_embedding [N, D], frame_tokens [N, S, 35, D] (window order), sel int32 [N] on the device: every per-env choice --
        mask, token gather, action-row gather -- is made on the device, so one CUDA graph serves every mix of fill levels.
        sample_noise [N, steps, 7] or None.  Returns (arm [N, steps, 6], gripper [N, steps, 1]), or the backbone's action-token
        rows [N, steps, D] with return_features.  At N = 1 the actions come from the fused sampler kernel (with
        FUSED_SAMPLER), at N >= 2 from the module sampler."""
        assert self.use_dit_head and self.action_pred_steps > 0
        N, S = frame_tokens.shape[:2]
        D = self.hidden_dim
        dev = frame_tokens.device
        assert S == self.sequence_length and sel.dtype == torch.int32 and sel.shape == (N,)
        stack, idx, r0 = self._batched_rollout_tables(dev)
        q = torch.cat([t.reshape(-1, D) for t in self._query_tokens()], dim=0)                    # [n_b, D]
        n_b = q.shape[0]
        n_tok = 1 + frame_tokens.shape[2] + n_b
        pos = self.transformer_backbone_position_embedding.view(1, S, 1, D)
        a_tok = torch.cat((text_embedding.view(N, 1, 1, D).expand(N, S, 1, D), frame_tokens), dim=2)   # [N, S, 36, D]
        full = (torch.cat((a_tok, q.view(1, 1, n_b, D).expand(N, S, n_b, D)), dim=2) + pos).reshape(N * S * n_tok, D)
        sel64 = sel.long()
        rows = idx.index_select(0, sel64) + (torch.arange(N, device=dev) * (S * n_tok)).unsqueeze(1)    # [N, Lb]
        x = full.index_select(0, rows.flatten()).view(N, -1, D)
        x = self.embedding_layer_norm(x.contiguous())
        h = self.transformer_backbone(inputs_embeds=x, attention_mask=stack.select(sel))
        arow = r0.index_select(0, sel64).unsqueeze(1) + torch.arange(self.action_pred_steps, device=dev)  # [N, steps]
        feat = h.gather(1, arow.unsqueeze(2).expand(N, self.action_pred_steps, D))                 # [N, steps, D]
        if return_features:
            return feat
        samples = self._ddim_actions(feat, sample_noise, dev)
        return samples[..., :6], samples[..., 6:]

    @torch.no_grad()
    def rollout_action(self, text_embedding, frame_tokens, sel, sample_noise=None, prune=True, return_features=False):
        """One action for the timestep `sel` of a window (mode='test' of `forward`, restricted to what that action needs).

        text_embedding [1, D] (encode_text_embedding), frame_tokens [S, 35, D] (encode_frame_tokens; frames after `sel`
        are the padded repeats of the reference wrapper and are ignored when prune=True).  Returns (arm [1, steps, 6],
        gripper [1, steps, 1]) == rows `sel` of the full-window outputs.
          prune=False: the backbone sees exactly the full window's L tokens (bit-identical activations for row `sel`);
          prune=True:  tokens that no kept row can attend to are dropped before the backbone (L=930 -> 36*(sel+1)+57 at the
                       eval.sh configuration); same mathematics, different KV tiling => equal up to bf16 rounding.
        The DiT / DDIM sampler only runs for the selected timestep (the reference samples all S and discards S-1)."""
        assert self.use_dit_head and self.action_pred_steps > 0
        S, D = self.sequence_length, self.hidden_dim
        dev = frame_tokens.device
        n_a = 1 + 1 + 2 * self.NUM_RESAMPLER_QUERY + 2
        q = torch.cat([t.reshape(-1, D) for t in self._query_tokens()], dim=0)                    # [n_b, D]
        n_b = q.shape[0]
        pos = self.transformer_backbone_position_embedding.view(S, 1, D)
        a_tok = torch.cat((text_embedding.view(1, 1, D).expand(S, 1, D), frame_tokens), dim=1)   # [S, 36, D]
        mask, idx, idx_host = self._rollout_mask(sel, prune, dev)
        full = (torch.cat((a_tok, q.unsqueeze(0).expand(S, n_b, D)), dim=1) + pos).reshape(S * (n_a + n_b), D)
        a0 = sel * (n_a + n_b) + n_a + n_b - self.action_pred_steps      # first action row of the selected timestep
        if prune:
            x = full.index_select(0, idx).unsqueeze(0)                   # kept tokens, original order
            r0 = int((idx_host < a0).sum())                                 # the action rows are kept: their new position
            act_rows = slice(r0, r0 + self.action_pred_steps)
        else:
            x = full.unsqueeze(0)
            act_rows = slice(a0, a0 + self.action_pred_steps)
        x = self.embedding_layer_norm(x.contiguous())
        h = self.transformer_backbone(inputs_embeds=x, attention_mask=mask)
        feat = h[:, act_rows, :].contiguous()                                                   # [1, steps, D]
        if return_features:                                    # the backbone's action-token rows (parity tests)
            return feat
        samples = self._ddim_actions(feat, sample_noise, dev)
        return samples[..., :6], samples[..., 6:]

    # ------------------------------------------------------------------------------------------------------------------
    def forward(self, image_primary, image_wrist, state, text_token, action=None, track_infos=None, action_label=None,
                mode="train", diffusion_noise=None, diffusion_timestep=None, diffusion_drop_ids=None, sample_noise=None):
        """Reference :609-991.  The four trailing keyword arguments inject the tensors the reference samples inside
        forward (action_model.py:59-60, models.py:83, dreamvla_model.py:944) so parity tests can line them up."""
        device_drop = self.training and self.redraws_mask and self.obs_drop_on_device
        if self.training and self.redraws_mask and not device_drop:
            # :610-628 mask regenerated each forward; only the np.random column drop (:55-59) makes it differ
            self.attention_mask = nn.Parameter(self._make_mask().to(self.attention_mask.device), requires_grad=False)
        B, S, _ = state.shape
        D = self.hidden_dim
        dev = image_primary.device
        dt = torch.bfloat16
        image_pred = depth_pred = traj_pred = dino_pred = sam_pred = None
        arm_pred_action = gripper_pred_action = None
        arm_pred_state = gripper_pred_state = loss_arm_action = None

        # ---- text (:643-653) ----
        with torch.no_grad():
            if text_token.stride(1) == 0 and S > 1:     # one sentence expanded over the window: encode once
                tf = self.clip_model.encode_text(text_token[:, 0].contiguous()).to(dt)
                text_feature = tf.unsqueeze(1).expand(B, S, -1).reshape(B * S, -1)
            else:
                text_feature = self.clip_model.encode_text(text_token.flatten(0, 1)).to(dt)
        text_embedding = self.text_projector(text_feature).view(B, S, -1, D)

        # ---- state (:656-664) and vision: both cameras in one batch (:666-673, :716-737) ----
        state_embedding = self._encode_state(state.flatten(0, 1)).view(B, S, -1, D)
        pe, we, cp, cw = self._encode_vision(image_primary.flatten(0, 1), image_wrist.flatten(0, 1))
        image_primary_embedding, image_wrist_embedding = pe.view(B, S, -1, D), we.view(B, S, -1, D)
        cls_p, cls_w = cp.view(B, S, -1, D), cw.view(B, S, -1, D)

        # ---- token assembly (:739-759); slot order is part of the contract ----
        # per timestep: [text . state . primary nq . wrist nq . cls_p . cls_w | obs . depth . dino . sam . traj | action]
        a_parts = [text_embedding, state_embedding, image_primary_embedding, image_wrist_embedding, cls_p, cls_w]
        q_parts = [t.expand(B, S, -1, -1) for t in self._query_tokens()]      # query slots, action slots last
        n_act = self.action_pred_steps if self.action_pred_steps > 0 else 0
        n_a = 1 + 1 + 2 * self.NUM_RESAMPLER_QUERY + 2
        n_q = sum(t.shape[2] for t in q_parts) - n_act
        transformer_input = torch.cat(a_parts + q_parts, dim=2)
        transformer_input = transformer_input + self.transformer_backbone_position_embedding
        transformer_input = transformer_input.flatten(1, 2)

        # ---- backbone (:765-790) ----
        transformer_input = self.embedding_layer_norm(transformer_input)
        marks = getattr(self, "_dvla_grad_marks", None)      # set by TrainStep: overlap the gradient all-reduce with backward
        self.transformer_backbone._dvla_grad_mark = marks["backbone_cuts"] if marks else None
        # device draw: one per forward, TrainStep advances the seed counter every micro-step (also under CUDA-graph replay)
        mask = self._device_obs_drop(dev).draw(ops.seed_counter(dev)) if device_drop else self._attn_mask(dev)
        transformer_output = self.transformer_backbone(inputs_embeds=transformer_input, attention_mask=mask)
        if marks and transformer_output.requires_grad:
            ops.on_grad_ready(transformer_output, marks["backbone_out"])
        transformer_output = transformer_output.view(B, S, -1, D)
        q_out = transformer_output[:, :, n_a:n_a + n_q]
        act_out = transformer_output[:, :, n_a + n_q:]

        # ---- world-knowledge heads (:793-911) ----
        cur = 0
        q4 = int(D / 4)
        if self.obs_pred and mode == "train":
            if self.share_query:
                feat = q_out[:, :, 0:self.NUM_OBS_TOKEN, :q4]
                cur = 0
            else:
                feat = q_out[:, :, 0:self.NUM_OBS_TOKEN, :]
                cur += self.NUM_OBS_TOKEN
            g = self.NUM_OBS_TOKEN // self.NUM_OBS_TOKEN_PER_IMAGE
            out = _WorldDecoder.run(feat, self.image_decoder_obs_pred_projector, self.mask_token,
                                    self.image_decoder_position_embedding, self.image_decoder, self.image_decoder_norm,
                                    self.image_decoder_pred, g, self.NUM_OBS_TOKEN_PER_IMAGE, self.NUM_MASK_TOKEN, D)
            image_pred = out.view(B * S, g, self.pred_num, self.NUM_MASK_TOKEN // self.pred_num, -1)
        if self.depth_pred and mode == "train":
            if self.share_query:
                feat = q_out[:, :, cur:cur + self.NUM_DEPTH_TOKEN, q4:2 * q4]
                cur = 0
            else:
                feat = q_out[:, :, cur:cur + self.NUM_DEPTH_TOKEN, :]
                cur += self.NUM_DEPTH_TOKEN
            g = self.NUM_DEPTH_TOKEN // self.NUM_OBS_TOKEN_PER_DEPTH
            out = _WorldDecoder.run(feat, self.depth_decoder_obs_pred_projector, self.depth_mask_token,
                                    self.depth_decoder_position_embedding, self.depth_decoder, self.depth_decoder_norm,
                                    self.depth_decoder_pred, g, self.NUM_OBS_TOKEN_PER_DEPTH, self.NUM_DEPTH_MASK_TOKEN, D,
                                    act="relu")                                             # F.relu (:842) fused
            depth_pred = out.view(B * S, g, self.pred_num, self.NUM_DEPTH_MASK_TOKEN // self.pred_num, -1)
        if self.dino_feat_pred and mode == "train":
            if self.share_query:
                feat = q_out[:, :, cur:cur + self.NUM_DINO_TOKEN, 2 * q4:3 * q4]
                cur = 0
            else:
                feat = q_out[:, :, cur:cur + self.NUM_DINO_TOKEN, :]
                cur += self.NUM_DINO_TOKEN
            g = self.NUM_DINO_TOKEN // self.NUM_OBS_TOKEN_PER_DINO
            out = _WorldDecoder.run(feat, self.dino_decoder_obs_pred_projector, self.dino_mask_token,
                                    self.dino_decoder_position_embedding, self.dino_feat_decoder, self.dino_decoder_norm,
                                    self.dino_decoder_pred, g, self.NUM_OBS_TOKEN_PER_DINO, self.NUM_DINO_MASK_TOKEN, D)
            dino_pred = out.view(B * S, g, self.pred_num, self.NUM_DINO_MASK_TOKEN // self.pred_num, -1)
        if self.sam_feat_pred and mode == "train":
            if self.share_query:
                feat = q_out[:, :, cur:cur + self.NUM_SAM_TOKEN, 3 * q4:D]
                cur = 0
            else:
                feat = q_out[:, :, cur:cur + self.NUM_SAM_TOKEN, :]
                cur += self.NUM_SAM_TOKEN
            g = self.NUM_SAM_TOKEN // self.NUM_OBS_TOKEN_PER_SAM
            out = _WorldDecoder.run(feat, self.sam_decoder_obs_pred_projector, self.sam_mask_token,
                                    self.sam_decoder_position_embedding, self.sam_feat_decoder, self.sam_decoder_norm,
                                    self.sam_decoder_pred, g, self.NUM_OBS_TOKEN_PER_SAM, self.NUM_SAM_MASK_TOKEN, D)
            sam_pred = out.view(B * S, g, self.pred_num, self.NUM_SAM_MASK_TOKEN // self.pred_num, -1)
        if self.trajectory_pred and mode == "train":
            feat = q_out[:, :, cur:cur + self.NUM_TRAJ_TOKEN, :]
            g = self.NUM_TRAJ_TOKEN // self.NUM_OBS_TOKEN_PER_TRAJ
            out = _WorldDecoder.run(feat, self.traj_decoder_obs_pred_projector, self.traj_mask_token,
                                    self.traj_decoder_position_embedding, self.traj_decoder, self.traj_decoder_norm,
                                    self.traj_decoder_pred, g, self.NUM_OBS_TOKEN_PER_TRAJ, self.NUM_TRAJ_MASK_TOKEN, D)
            traj_pred = out.view(B * S, g, self.pred_num, self.NUM_TRAJ_MASK_TOKEN // self.pred_num, -1)
            cur += self.NUM_TRAJ_TOKEN

        # ---- action head (:915-987) ----
        if self.action_pred_steps > 0:
            action_pred_feature = act_out
            if not self.use_dit_head:
                h = self.action_decoder[0](action_pred_feature, act="relu")
                h = self.action_decoder[2](h, act="relu")
                arm_pred_action = torch.tanh(self.arm_action_decoder[0](h).float()).to(dt)
                gripper_pred_action = torch.sigmoid(self.gripper_action_decoder[0](h).float()).to(dt)
            elif mode == "train":
                feat = action_pred_feature[:, :self.sequence_length - self.atten_goal].flatten(0, 1)
                labels = action_label.flatten(0, 1).to(dt)
                rep = 8
                arm_pred_action = self.action_model.loss(labels.repeat(rep, 1, 1), feat.repeat(rep, 1, 1),
                                                         noise=diffusion_noise, timestep=diffusion_timestep,
                                                         force_drop_ids=diffusion_drop_ids)
                gripper_pred_action = arm_pred_action
            else:  # mode == 'test': 10-step DDIM with classifier-free guidance 1.5 (:935-987)
                samples = self._ddim_actions(action_pred_feature.flatten(0, 1), sample_noise, dev)
                arm_pred_action, gripper_pred_action = samples.unsqueeze(0)[..., :6], samples.unsqueeze(0)[..., 6:]
        return (arm_pred_action, gripper_pred_action, image_pred, arm_pred_state, gripper_pred_state, loss_arm_action,
                depth_pred, traj_pred, dino_pred, sam_pred)
