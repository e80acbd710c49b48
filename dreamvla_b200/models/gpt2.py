"""Trimmed GPT-2 backbone on sm_90a kernels -- mirror of reference models/gpt2.py:22-480.

Takes `inputs_embeds` [B, L, D] and the additive {0,-inf} attention mask of dreamvla_model.py:25-66; both
`attn_implementation` values of the reference ("eager" gpt2.py:61-84, "sdpa" gpt2.py:196-284) map to the same
bit-mask flash kernel.  Parameter names/layouts follow HF (h.N.ln_1, attn.c_attn [D,3D] (in,out), attn.c_proj,
ln_2, mlp.c_fc, mlp.c_proj, ln_f).  Dropouts (embd/attn/resid, GPT2Config defaults 0.1) run inside the kernels
(GEMM epilogue, attention probabilities) with a counter-based RNG.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch
import torch.nn as nn

from .. import ops
from .layers import Conv1D, LayerNorm


@dataclass
class GPT2Config:  # the subset of transformers.GPT2Config the reference reads (dreamvla_model.py:301-307)
    hidden_size: int = 768
    n_layer: int = 12
    n_head: int = 12
    n_inner: int | None = None
    vocab_size: int = 1
    activation_function: str = "gelu_new"
    resid_pdrop: float = 0.1
    embd_pdrop: float = 0.1
    attn_pdrop: float = 0.1
    layer_norm_epsilon: float = 1e-5
    initializer_range: float = 0.02
    scale_attn_weights: bool = True
    attn_implementation: object = "sdpa"
    max_position_embeddings: int = 1024

    @property
    def num_hidden_layers(self):
        return self.n_layer

    @property
    def num_attention_heads(self):
        return self.n_head


class GPT2Attention(nn.Module):
    def __init__(self, config, layer_idx=None):
        super().__init__()
        self.embed_dim = config.hidden_size
        self.num_heads = config.num_attention_heads
        self.head_dim = self.embed_dim // self.num_heads
        assert self.head_dim == 64, "dreamvla_b200 attention kernels need head_dim == 64"
        self.c_attn = Conv1D(3 * self.embed_dim, self.embed_dim)
        self.c_proj = Conv1D(self.embed_dim, self.embed_dim)
        self.attn_pdrop = config.attn_pdrop
        self.resid_pdrop = config.resid_pdrop
        self.scale = 1.0 / math.sqrt(self.head_dim) if config.scale_attn_weights else 1.0

    def forward(self, hidden_states, attn_mask, residual):
        B, Lq, D = hidden_states.shape
        qkv = self.c_attn(hidden_states).view(B, Lq, 3, self.num_heads, self.head_dim)
        o = ops.self_attention_fused(qkv, self.scale, attn_mask, self.attn_pdrop if self.training else 0.0)
        return self.c_proj(o.view(B, Lq, D), residual=residual, dropout_p=self.resid_pdrop if self.training else 0.0)


GPT2SdpaAttention = GPT2Attention


class GPT2MLP(nn.Module):
    def __init__(self, intermediate_size, config):
        super().__init__()
        self.c_fc = Conv1D(intermediate_size, config.hidden_size)
        self.c_proj = Conv1D(config.hidden_size, intermediate_size)
        self.act = config.activation_function
        self.resid_pdrop = config.resid_pdrop

    def forward(self, hidden_states, residual):
        return ops.mlp(hidden_states, self.c_fc.weight, self.c_fc.bias, self.c_proj.weight, self.c_proj.bias, act=self.act,
                       residual=residual, weight_kn=True, dropout_p=self.resid_pdrop if self.training else 0.0)


class GPT2Block(nn.Module):
    def __init__(self, config, layer_idx=None):
        super().__init__()
        inner = config.n_inner if config.n_inner is not None else 4 * config.hidden_size
        self.ln_1 = LayerNorm(config.hidden_size, eps=config.layer_norm_epsilon)
        self.attn = GPT2Attention(config, layer_idx)
        self.ln_2 = LayerNorm(config.hidden_size, eps=config.layer_norm_epsilon)
        self.mlp = GPT2MLP(inner, config)

    def forward(self, hidden_states, attn_mask):
        res, normed = self.ln_1.fork(hidden_states)          # the two gradients of x are summed inside LayerNorm-backward
        hidden_states = self.attn(normed, attn_mask, residual=res)
        res, normed = self.ln_2.fork(hidden_states)
        return self.mlp(normed, residual=res)


class GPT2Model(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.embed_dim = config.hidden_size
        self.embd_pdrop = config.embd_pdrop
        self.h = nn.ModuleList([GPT2Block(config, layer_idx=i) for i in range(config.num_hidden_layers)])
        self.ln_f = LayerNorm(self.embed_dim, eps=config.layer_norm_epsilon)
        self.apply(self._init_weights)

    def _init_weights(self, module):  # gpt2.py:359-384
        if isinstance(module, (nn.Linear, Conv1D)):
            module.weight.data.normal_(mean=0.0, std=self.config.initializer_range)
            if module.bias is not None:
                module.bias.data.zero_()
        elif isinstance(module, nn.LayerNorm):
            module.bias.data.zero_()
            module.weight.data.fill_(1.0)
        for name, p in module.named_parameters():
            if name == "c_proj.weight":
                p.data.normal_(mean=0.0, std=(self.config.initializer_range / math.sqrt(2 * self.config.n_layer)))

    def forward(self, attention_mask=None, inputs_embeds=None):
        """attention_mask: ops.AttnMask (preferred) or the reference's additive float mask [L,L] / [B,1,L,L]."""
        mask = attention_mask
        if isinstance(mask, torch.Tensor):
            m2 = mask[0, 0] if mask.dim() == 4 else mask
            mask = ops.AttnMask.from_additive(m2, inputs_embeds.device)
        h = ops.dropout(inputs_embeds, self.embd_pdrop, self.training)
        marks = dict(getattr(self, "_dvla_grad_mark", None) or ())   # {layer index: callback}: see TrainStep._arm_overlap
        for i, block in enumerate(self.h):
            if i in marks and h.requires_grad:
                ops.on_grad_ready(h, marks[i])               # fires when layers >= i have finished their backward
            h = block(h, mask)
        return self.ln_f(h)
