"""CLIP text tower (openai/CLIP model.py `encode_text`, ViT-B/32 text hyper-parameters) on sm_90a kernels.

Boundary input of the hot path (dreamvla_model.py:643-649; SURVEY §2.3 k17): frozen, no_grad.  openai/CLIP is not
installable offline, so `load()` returns a random-initialised tower with CLIP's parameter names
(token_embedding, positional_embedding, transformer.resblocks.N.{ln_1, attn.in_proj_weight/bias, attn.out_proj,
ln_2, mlp.c_fc, mlp.c_proj}, ln_final, text_projection) so that a real CLIP state_dict loads with strict=False.
Exact win kept from SURVEY k17: a sentence repeated over the window (text_token expanded along S, as both the train
loop and the rollout wrappers do) is encoded once by DreamVLA.forward (the reference encodes it S times).
"""
from __future__ import annotations

from collections import OrderedDict

import torch
import torch.nn as nn

from .. import ops
from .layers import LayerNorm, Linear


class _InProjAttention(nn.Module):
    """Parameter container matching nn.MultiheadAttention's names."""

    def __init__(self, d_model, n_head):
        super().__init__()
        self.in_proj_weight = nn.Parameter(torch.empty(3 * d_model, d_model))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * d_model))
        self.out_proj = Linear(d_model, d_model)
        self.n_head = n_head


class _QuickGELU(nn.Module):
    def forward(self, x):
        return x


class ResidualAttentionBlock(nn.Module):
    def __init__(self, d_model, n_head):
        super().__init__()
        self.attn = _InProjAttention(d_model, n_head)
        self.ln_1 = LayerNorm(d_model)
        self.mlp = nn.Sequential(OrderedDict([("c_fc", Linear(d_model, d_model * 4)), ("gelu", _QuickGELU()),
                                              ("c_proj", Linear(d_model * 4, d_model))]))
        self.ln_2 = LayerNorm(d_model)

    def forward(self, x, mask):
        B, T, D = x.shape
        H = self.attn.n_head
        qkv = ops.linear(self.ln_1(x), self.attn.in_proj_weight, self.attn.in_proj_bias).view(B, T, 3, H, D // H)
        o = ops.self_attention_fused(qkv, (D // H) ** -0.5, mask)
        x = self.attn.out_proj(o.view(B, T, D), residual=x)
        h = self.mlp.c_fc(self.ln_2(x), act="quick_gelu")
        return self.mlp.c_proj(h, residual=x)


class _Transformer(nn.Module):
    def __init__(self, width, layers, heads):
        super().__init__()
        self.width, self.layers = width, layers
        self.resblocks = nn.ModuleList([ResidualAttentionBlock(width, heads) for _ in range(layers)])


class CLIPTextTower(nn.Module):
    def __init__(self, embed_dim=512, context_length=77, vocab_size=49408, width=512, heads=8, layers=12):
        super().__init__()
        assert width // heads == 64
        self.context_length = context_length
        self.transformer = _Transformer(width, layers, heads)
        self.token_embedding = nn.Embedding(vocab_size, width)
        self.positional_embedding = nn.Parameter(torch.empty(context_length, width))
        self.ln_final = LayerNorm(width)
        self.text_projection = nn.Parameter(torch.empty(width, embed_dim))
        self.logit_scale = nn.Parameter(torch.ones([]) * 2.6592)
        self._mask = None
        nn.init.normal_(self.token_embedding.weight, std=0.02)
        nn.init.normal_(self.positional_embedding, std=0.01)
        proj_std = (width ** -0.5) * ((2 * layers) ** -0.5)
        for blk in self.transformer.resblocks:
            nn.init.normal_(blk.attn.in_proj_weight, std=width ** -0.5)
            nn.init.normal_(blk.attn.out_proj.weight, std=proj_std)
            nn.init.normal_(blk.mlp.c_fc.weight, std=(2 * width) ** -0.5)
            nn.init.normal_(blk.mlp.c_proj.weight, std=proj_std)
        nn.init.normal_(self.text_projection, std=width ** -0.5)

    @property
    def dtype(self):
        return self.token_embedding.weight.dtype

    @torch.no_grad()
    def encode_text(self, text):
        """text int [n, 77] -> [n, embed_dim].  (No host sync: CUDA-graph capturable.)"""
        uniq = text
        x = self.token_embedding(uniq) + self.positional_embedding
        if self._mask is None or self._mask.bits.device != x.device:
            self._mask = ops.AttnMask.causal(self.context_length, x.device)
        for blk in self.transformer.resblocks:
            x = blk(x, self._mask)
        x = self.ln_final(x)
        eot = x[torch.arange(x.shape[0], device=x.device), uniq.argmax(dim=-1)]
        return ops.linear(eot, self.text_projection, None, weight_kn=True)


def load(name="ViT-B/32", device="cpu", seed=20240607):
    """Stand-in for clip.load (dreamvla_model.py:511-514): (model, preprocess)."""
    state = torch.random.get_rng_state()
    torch.manual_seed(seed)
    model = CLIPTextTower()
    torch.random.set_rng_state(state)
    return model.to(device), (lambda img: img)
