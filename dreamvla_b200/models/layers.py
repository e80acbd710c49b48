"""Building blocks with the parameter names / shapes of the reference's third-party layers, forward on sm_90a kernels.

  Linear      == torch.nn.Linear            (weight [out,in])              -> ops.linear (wgmma GEMM + fused epilogue)
  Conv1D      == transformers Conv1D        (weight [in,out], gpt2.py:53)  -> ops.linear(weight_kn=True)
  LayerNorm   == torch.nn.LayerNorm                                        -> ops.layer_norm
  Attention / Mlp / Block == timm 0.9.16 vision_transformer.{Attention, Mlp, Block} (names norm1, attn.qkv, attn.proj,
                norm2, mlp.fc1, mlp.fc2) used by vit_mae.py:73-75, dreamvla_model.py:348-433, action_model/models.py:130-134

Subclassing nn.Linear / nn.LayerNorm keeps `isinstance` based initialisers (dreamvla_model.py:581-591) working unchanged.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import ops


def _require_bf16(p: torch.Tensor, what: str):
    if p.dtype != torch.bfloat16 or not p.is_cuda:
        raise RuntimeError(
            f"{what}: dreamvla_b200 kernels are bf16/CUDA only (got {p.dtype} on {p.device}); cast the model with "
            ".bfloat16() and move it to an H100 -- there is no CPU or fp32 fallback path")


class Linear(nn.Linear):
    def forward(self, x, act=None, residual=None, dropout_p=0.0):
        _require_bf16(self.weight, "Linear")
        return ops.linear(x, self.weight, self.bias, act=act, residual=residual, dropout_p=dropout_p)


class Conv1D(nn.Module):
    """HF Conv1D: y = x @ W + b with W [nx, nf] (in, out)."""

    def __init__(self, nf, nx):
        super().__init__()
        self.nf = nf
        self.weight = nn.Parameter(torch.empty(nx, nf))
        self.bias = nn.Parameter(torch.zeros(nf))
        nn.init.normal_(self.weight, std=0.02)

    def forward(self, x, act=None, residual=None, dropout_p=0.0):
        _require_bf16(self.weight, "Conv1D")
        return ops.linear(x, self.weight, self.bias, act=act, residual=residual, weight_kn=True, dropout_p=dropout_p)


class LayerNorm(nn.LayerNorm):
    def forward(self, x):
        if self.weight is not None:
            _require_bf16(self.weight, "LayerNorm")
        return ops.layer_norm(x, self.weight, self.bias, self.eps)

    def fork(self, x):
        """(x, LayerNorm(x)) with both gradients of x summed inside the LayerNorm-backward kernel (pre-norm residual blocks)."""
        if self.weight is not None:
            _require_bf16(self.weight, "LayerNorm")
        return ops.layer_norm_fork(x, self.weight, self.bias, self.eps)


class Attention(nn.Module):
    """timm Attention (fused qkv Linear, SDPA, proj); head_dim 64, or 96 on short sequences (the DiT-S action head)."""

    def __init__(self, dim, num_heads=8, qkv_bias=False):
        super().__init__()
        assert dim % num_heads == 0 and dim // num_heads in (64, 96), \
            "dreamvla_b200 attention kernels need head_dim 64, or 96 on short sequences (Lq <= 32, Lk <= 64)"
        self.num_heads = num_heads
        self.head_dim = dim // num_heads
        self.scale = self.head_dim ** -0.5
        self.qkv = Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = Linear(dim, dim)

    def forward(self, x, residual=None):
        B, N, C = x.shape
        qkv = self.qkv(x).view(B, N, 3, self.num_heads, self.head_dim)
        o = ops.self_attention_fused(qkv, self.scale)
        return self.proj(o.view(B, N, C), residual=residual)


class Mlp(nn.Module):
    def __init__(self, in_features, hidden_features, act="gelu_erf"):
        super().__init__()
        self.fc1 = Linear(in_features, hidden_features)
        self.fc2 = Linear(hidden_features, in_features)
        self.act = act

    def forward(self, x, residual=None):
        _require_bf16(self.fc1.weight, "Mlp")
        return ops.mlp(x, self.fc1.weight, self.fc1.bias, self.fc2.weight, self.fc2.bias, act=self.act, residual=residual)


class Block(nn.Module):
    """timm Block: x + attn(norm1 x); x + mlp(norm2 x).  Residual adds are fused into the proj / fc2 GEMM epilogues."""

    def __init__(self, dim, num_heads, mlp_ratio=4.0, qkv_bias=False, norm_layer=None, act="gelu_erf", eps=1e-5,
                 elementwise_affine=True):
        super().__init__()
        mk = norm_layer if norm_layer is not None else (lambda d: LayerNorm(d, eps=eps, elementwise_affine=elementwise_affine))
        self.norm1 = mk(dim)
        self.attn = Attention(dim, num_heads=num_heads, qkv_bias=qkv_bias)
        self.norm2 = mk(dim)
        self.mlp = Mlp(dim, int(dim * mlp_ratio), act=act)

    def forward(self, x):
        if isinstance(self.norm1, LayerNorm) and isinstance(self.norm2, LayerNorm):
            res, n = self.norm1.fork(x)
            x = self.attn(n, residual=res)
            res, n = self.norm2.fork(x)
            return self.mlp(n, residual=res)
        x = self.attn(self.norm1(x), residual=x)
        return self.mlp(self.norm2(x), residual=x)
