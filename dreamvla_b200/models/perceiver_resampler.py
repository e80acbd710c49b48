"""Flamingo Perceiver resampler on sm_90a kernels -- mirror of reference models/perceiver_resampler.py:11-128.

Parameter names follow the reference (layers.N.0.{norm_media,norm_latents,to_q,to_kv,to_out}, layers.N.1.{0,1,3}, norm).
Cross-attention over [media ; latents] keys runs in the flash kernel (no materialised `sim`, perceiver_resampler.py:55-57);
`q * scale` and the amax subtraction are folded into the kernel's scaled, max-subtracted online softmax.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import ops
from .layers import LayerNorm, Linear


class _GELU(nn.Module):  # placeholder keeping nn.Sequential indices (0: LN, 1: Linear, 2: GELU, 3: Linear)
    def forward(self, x):
        return x


def FeedForward(dim, mult=4):
    inner_dim = int(dim * mult)
    return nn.Sequential(LayerNorm(dim), Linear(dim, inner_dim, bias=False), _GELU(), Linear(inner_dim, dim, bias=False))


class PerceiverAttention(nn.Module):
    def __init__(self, *, dim, dim_head=64, heads=8):
        super().__init__()
        assert dim_head == 64, "dreamvla_b200 attention kernels need head_dim == 64"
        self.scale = dim_head ** -0.5
        self.heads = heads
        inner_dim = dim_head * heads
        self.norm_media = LayerNorm(dim)
        self.norm_latents = LayerNorm(dim)
        self.to_q = Linear(dim, inner_dim, bias=False)
        self.to_kv = Linear(dim, inner_dim * 2, bias=False)
        self.to_out = Linear(inner_dim, dim, bias=False)

    def forward(self, x, latents):
        """x [n, v, D] media, latents [n, nq, D] -> to_out(attn) + latents (residual fused)."""
        n, v, D = x.shape
        nq = latents.shape[1]
        h = self.heads
        xn = self.norm_media(x)
        ln = self.norm_latents(latents)
        q = self.to_q(ln).view(n, nq, h, 64)
        kv = self.to_kv(torch.cat((xn, ln), dim=1)).view(n, v + nq, 2, h, 64)
        o = ops.attention(q, kv[:, :, 0], kv[:, :, 1], self.scale)
        return self.to_out(o.view(n, nq, h * 64), residual=latents)


class PerceiverResampler(nn.Module):
    def __init__(self, *, dim, depth=6, dim_head=64, heads=8, num_latents=64, max_num_media=None, max_num_frames=None,
                 ff_mult=4):
        super().__init__()
        if max_num_media is not None or max_num_frames is not None:
            raise NotImplementedError("frame/media time embeddings are not used by DreamVLA (dreamvla_model.py:218)")
        self.latents = nn.Parameter(torch.randn(num_latents, dim))
        self.layers = nn.ModuleList([nn.ModuleList([PerceiverAttention(dim=dim, dim_head=dim_head, heads=heads),
                                                    FeedForward(dim=dim, mult=ff_mult)]) for _ in range(depth)])
        self.norm = LayerNorm(dim)

    def forward(self, x):
        """x [b, T, F, v, D] -> [b, T, n, D]  (perceiver_resampler.py:103-128)."""
        b, T, F, v, D = x.shape
        x = x.reshape(b * T, F * v, D)
        latents = self.latents.unsqueeze(0).expand(b * T, -1, -1).contiguous()
        for attn, ff in self.layers:
            latents = attn(x, latents)
            latents = ops.mlp(ff[0](latents), ff[1].weight, None, ff[3].weight, None, act="gelu_erf", residual=latents)
        return self.norm(latents).view(b, T, -1, D)
