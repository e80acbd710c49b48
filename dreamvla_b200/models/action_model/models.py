"""DiT action head on sm_90a kernels -- mirror of reference models/action_model/models.py:28-268.

Plain pre-LN ViT blocks (no adaLN): LayerNorm without affine (eps 1e-6), timm Attention (qkv_bias), Mlp with
GELU(tanh).  Parameter names follow the reference (x_embedder.linear, t_embedder.mlp.{0,2}, z_embedder.{linear,
uncondition}, positional_embedding, blocks.N.{attn.qkv, attn.proj, mlp.fc1, mlp.fc2}, final_layer.linear,
history_embedder.linear).
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from ..layers import Block, LayerNorm, Linear


class _SiLU(nn.Module):
    def forward(self, x):
        return x


class TimestepEmbedder(nn.Module):
    def __init__(self, hidden_size, frequency_embedding_size=256):
        super().__init__()
        self.mlp = nn.Sequential(Linear(frequency_embedding_size, hidden_size, bias=True), _SiLU(),
                                 Linear(hidden_size, hidden_size, bias=True))
        self.frequency_embedding_size = frequency_embedding_size

    @staticmethod
    def timestep_embedding(t, dim, max_period=10000):  # models.py:43-60 (fp32)
        half = dim // 2
        freqs = torch.exp(-math.log(max_period) * torch.arange(start=0, end=half, dtype=torch.float32, device=t.device) / half)
        args = t[:, None].float() * freqs[None]
        embedding = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
        if dim % 2:
            embedding = torch.cat([embedding, torch.zeros_like(embedding[:, :1])], dim=-1)
        return embedding

    def forward(self, t):
        t_freq = self.timestep_embedding(t, self.frequency_embedding_size).to(self.mlp[0].weight.dtype)
        return self.mlp[2](self.mlp[0](t_freq, act="silu"))


class LabelEmbedder(nn.Module):
    def __init__(self, in_size, hidden_size, dropout_prob=0.1, conditions_shape=(1, 1, 384)):
        super().__init__()
        self.linear = Linear(in_size, hidden_size)
        self.dropout_prob = dropout_prob
        if dropout_prob > 0:
            self.uncondition = nn.Parameter(torch.empty(conditions_shape[1:]))

    def token_drop(self, conditions, force_drop_ids=None):  # models.py:78-87
        if force_drop_ids is None:
            drop_ids = torch.rand(conditions.shape[0], device=conditions.device) < self.dropout_prob
        else:
            drop_ids = force_drop_ids == 1
        return torch.where(drop_ids.unsqueeze(1).unsqueeze(1).expand(conditions.shape[0], *self.uncondition.shape),
                           self.uncondition, conditions)

    def forward(self, conditions, train, force_drop_ids=None):
        if (train and self.dropout_prob > 0) or (force_drop_ids is not None):
            conditions = self.token_drop(conditions, force_drop_ids)
        return self.linear(conditions)


class _LinearHolder(nn.Module):
    def __init__(self, action_size, hidden_size):
        super().__init__()
        self.linear = Linear(action_size, hidden_size)

    def forward(self, x):
        return self.linear(x)


ActionEmbedder = _LinearHolder
HistoryEmbedder = _LinearHolder


class DiTBlock(Block):
    def __init__(self, hidden_size, num_heads, mlp_ratio=4.0):
        super().__init__(hidden_size, num_heads, mlp_ratio, qkv_bias=True, act="gelu_tanh", eps=1e-6,
                         elementwise_affine=False)


class FinalLayer(nn.Module):
    def __init__(self, hidden_size, out_channels):
        super().__init__()
        self.norm_final = LayerNorm(hidden_size, elementwise_affine=False, eps=1e-6)
        self.linear = Linear(hidden_size, out_channels, bias=True)

    def forward(self, x):
        return self.linear(self.norm_final(x))


class DiT(nn.Module):
    def __init__(self, in_channels=7, hidden_size=1152, depth=28, num_heads=16, mlp_ratio=4.0, class_dropout_prob=0.1,
                 token_size=4096, future_action_window_size=1, past_action_window_size=0, learn_sigma=False):
        super().__init__()
        assert past_action_window_size == 0, "Error: action_history is not used now"
        assert not learn_sigma
        self.learn_sigma = learn_sigma
        self.in_channels = in_channels
        self.out_channels = in_channels
        self.class_dropout_prob = class_dropout_prob
        self.num_heads = num_heads
        self.past_action_window_size = past_action_window_size
        self.future_action_window_size = future_action_window_size
        self.history_embedder = HistoryEmbedder(action_size=in_channels, hidden_size=hidden_size)
        self.x_embedder = ActionEmbedder(action_size=in_channels, hidden_size=hidden_size)
        self.t_embedder = TimestepEmbedder(hidden_size)
        self.z_embedder = LabelEmbedder(in_size=token_size, hidden_size=hidden_size, dropout_prob=class_dropout_prob,
                                        conditions_shape=(1, 1, token_size))
        scale = hidden_size ** -0.5
        self.positional_embedding = nn.Parameter(
            scale * torch.randn(future_action_window_size + past_action_window_size + 1 + future_action_window_size + 1, hidden_size))
        self.blocks = nn.ModuleList([DiTBlock(hidden_size, num_heads, mlp_ratio=mlp_ratio) for _ in range(depth)])
        self.final_layer = FinalLayer(hidden_size, self.out_channels)
        self.initialize_weights()

    def initialize_weights(self):  # models.py:205-232
        def _basic_init(module):
            if isinstance(module, nn.Linear):
                torch.nn.init.xavier_uniform_(module.weight)
                if module.bias is not None:
                    nn.init.constant_(module.bias, 0)
        self.apply(_basic_init)
        nn.init.normal_(self.x_embedder.linear.weight, std=0.02)
        nn.init.constant_(self.x_embedder.linear.bias, 0)
        nn.init.normal_(self.history_embedder.linear.weight, std=0.02)
        nn.init.constant_(self.history_embedder.linear.bias, 0)
        if self.class_dropout_prob > 0:
            nn.init.normal_(self.z_embedder.uncondition, std=0.02)
        nn.init.normal_(self.z_embedder.linear.weight, std=0.02)
        nn.init.constant_(self.z_embedder.linear.bias, 0)
        nn.init.normal_(self.t_embedder.mlp[0].weight, std=0.02)
        nn.init.normal_(self.t_embedder.mlp[2].weight, std=0.02)
        nn.init.constant_(self.final_layer.linear.weight, 0)
        nn.init.constant_(self.final_layer.linear.bias, 0)

    def forward(self, x, t, z, force_drop_ids=None):
        """models.py:234-251.  x (N,T,7), t (N,), z (N,Tz,token) -> (N,T,7)."""
        dt = self.x_embedder.linear.weight.dtype
        x = self.x_embedder(x.to(dt))
        t = self.t_embedder(t)
        z = self.z_embedder(z.to(dt), self.training, force_drop_ids)
        c = t.unsqueeze(1) + z
        x = torch.cat((c, x), dim=1)
        x = x + self.positional_embedding
        for block in self.blocks:
            x = block(x)
        x = self.final_layer(x)
        return x[:, c.shape[1]:, :]

    def forward_with_cfg(self, x, t, z, cfg_scale):
        """models.py:253-268."""
        half = x[: len(x) // 2]
        combined = torch.cat([half, half], dim=0)
        model_out = self.forward(combined, t, z)
        eps, rest = model_out[:, :, :self.in_channels], model_out[:, :, self.in_channels:]
        cond_eps, uncond_eps = torch.split(eps, len(eps) // 2, dim=0)
        half_eps = uncond_eps + cfg_scale * (cond_eps - uncond_eps)
        eps = torch.cat([half_eps, half_eps], dim=0)
        return torch.cat([eps, rest], dim=2)
