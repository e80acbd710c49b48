"""MAE ViT-B/16 encoder on sm_90a kernels -- mirror of reference models/vit_mae.py:55-206 (encoder half only).

Only `forward_encoder(x, mask_ratio=0.0)` is on the hot path (dreamvla_model.py:672-673).  The MAE decoder half of the
reference class (26 M parameters, never executed by DreamVLA) is not instantiated; MAE checkpoints load with
strict=False exactly as in the reference (dreamvla_model.py:477-478).

Patch embedding (timm PatchEmbed = Conv2d k=s=16, vit_mae.py:66,188) is a GEMM over the im2col view
[N*196, 3*16*16] with bias + positional embedding fused in the epilogue (residual operand).

random_masking(x, 0.0) (vit_mae.py:157-182,194) keeps all 196 tokens but in a random order.  All consumers of the
patch tokens are permutation-invariant (ViT blocks are equivariant, PerceiverAttention sums over keys), so the
permutation is skipped here; outputs are identical in exact arithmetic (tests/test_oracle_cpu.py pins this on the
reference itself).
"""
from __future__ import annotations

from functools import partial

import numpy as np
import torch
import torch.nn as nn

from .. import ops
from .layers import Block, LayerNorm, _require_bf16


def get_1d_sincos_pos_embed_from_grid(embed_dim, pos):
    assert embed_dim % 2 == 0
    omega = np.arange(embed_dim // 2, dtype=np.float32)
    omega /= embed_dim / 2.0
    omega = 1.0 / 10000 ** omega
    out = np.einsum("m,d->md", pos.reshape(-1), omega)
    return np.concatenate([np.sin(out), np.cos(out)], axis=1)


def get_2d_sincos_pos_embed(embed_dim, grid_size, cls_token=False):
    """vit_mae.py:19-36 / dreamvla_model.py:101-116 (w goes first in the meshgrid)."""
    grid_h = np.arange(grid_size, dtype=np.float32)
    grid_w = np.arange(grid_size, dtype=np.float32)
    grid = np.stack(np.meshgrid(grid_w, grid_h), axis=0).reshape([2, 1, grid_size, grid_size])
    emb_h = get_1d_sincos_pos_embed_from_grid(embed_dim // 2, grid[0])
    emb_w = get_1d_sincos_pos_embed_from_grid(embed_dim // 2, grid[1])
    pos_embed = np.concatenate([emb_h, emb_w], axis=1)
    if cls_token:
        pos_embed = np.concatenate([np.zeros([1, embed_dim]), pos_embed], axis=0)
    return pos_embed


class PatchEmbed(nn.Module):
    """timm PatchEmbed parameter layout: proj.weight [E, C, p, p], proj.bias [E]."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768):
        super().__init__()
        self.img_size = (img_size, img_size)
        self.patch_size = (patch_size, patch_size)
        self.grid_size = (img_size // patch_size, img_size // patch_size)
        self.num_patches = self.grid_size[0] * self.grid_size[1]
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)  # parameters only

    def forward(self, x, pos_rows=None):
        """x [N, C, H, W] -> [N, num_patches, E]; pos_rows [N*num_patches, E] is added in the GEMM epilogue."""
        _require_bf16(self.proj.weight, "PatchEmbed")
        N, C, H, W = x.shape
        p = self.patch_size[0]
        gh, gw = H // p, W // p
        cols = x.view(N, C, gh, p, gw, p).permute(0, 2, 4, 1, 3, 5).reshape(N * gh * gw, C * p * p)
        w2 = self.proj.weight.view(self.proj.weight.shape[0], -1)
        y = ops.linear(cols, w2, self.proj.bias, residual=pos_rows)
        return y.view(N, gh * gw, -1)


class MaskedAutoencoderViT(nn.Module):
    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=1024, depth=24, num_heads=16,
                 decoder_embed_dim=512, decoder_depth=8, decoder_num_heads=16, mlp_ratio=4.0,
                 norm_layer=partial(LayerNorm, eps=1e-6), norm_pix_loss=False):
        super().__init__()
        self.patch_embed = PatchEmbed(img_size, patch_size, in_chans, embed_dim)
        num_patches = self.patch_embed.num_patches
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.pos_embed = nn.Parameter(torch.zeros(1, num_patches + 1, embed_dim), requires_grad=False)
        self.blocks = nn.ModuleList([Block(embed_dim, num_heads, mlp_ratio, qkv_bias=True, norm_layer=norm_layer)
                                     for _ in range(depth)])
        self.norm = norm_layer(embed_dim)
        self._pos_cache = None
        self.initialize_weights()

    def initialize_weights(self):  # vit_mae.py:103-133 (encoder part)
        pos_embed = get_2d_sincos_pos_embed(self.pos_embed.shape[-1], int(self.patch_embed.num_patches ** 0.5), cls_token=True)
        self.pos_embed.data.copy_(torch.from_numpy(pos_embed).float().unsqueeze(0))
        w = self.patch_embed.proj.weight.data
        torch.nn.init.xavier_uniform_(w.view([w.shape[0], -1]))
        torch.nn.init.normal_(self.cls_token, std=0.02)
        self.apply(self._init_weights)

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            torch.nn.init.xavier_uniform_(m.weight)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def _pos_rows(self, n_img):
        """pos_embed[:, 1:] repeated per image (the residual operand of the patch-embed GEMM), cached PER BATCH SIZE: a
        captured CUDA graph keeps the raw pointer of the tensor it saw, so an entry must outlive other batch sizes being
        used in between (rollout wrappers run 2-image and 2S-image batches through the same model)."""
        key = (n_img, self.pos_embed.data_ptr(), self.pos_embed._version)
        if self._pos_cache is None:
            self._pos_cache = {}
        rows = self._pos_cache.get(key)
        if rows is None:
            stale = [k for k in self._pos_cache if k[1:] != key[1:]]        # the parameter itself changed: graphs are stale too
            for k in stale:
                del self._pos_cache[k]
            rows = self._pos_cache[key] = self.pos_embed[0, 1:, :].repeat(n_img, 1).contiguous()
        return rows

    def forward_encoder(self, x, mask_ratio=0.0):
        """vit_mae.py:184-206 with mask_ratio == 0 (the only value DreamVLA uses)."""
        if mask_ratio != 0.0:
            raise NotImplementedError("dreamvla_b200 implements the DreamVLA hot path: mask_ratio must be 0.0")
        x = self.patch_embed(x, self._pos_rows(x.shape[0]))          # + pos_embed[:, 1:] fused
        cls = (self.cls_token + self.pos_embed[:, :1, :]).expand(x.shape[0], -1, -1)
        x = torch.cat((cls, x), dim=1)
        for blk in self.blocks:
            x = blk(x)
        return self.norm(x), None, None
