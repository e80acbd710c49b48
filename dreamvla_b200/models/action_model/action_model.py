"""ActionModel (DiT + IDDPM diffusion) and ActionModelFM (DiT + flow matching, `--use_fm`) -- mirror of reference
models/action_model/action_model.py:13-83 and :86-169."""
from __future__ import annotations

import torch
from torch import nn

from .gaussian_diffusion import FMDiffusion, create_diffusion, get_named_beta_schedule
from .models import DiT


def DiT_S(**kwargs):
    return DiT(depth=6, hidden_size=384, num_heads=4, **kwargs)


def DiT_B(**kwargs):
    return DiT(depth=12, hidden_size=768, num_heads=12, **kwargs)


def DiT_L(**kwargs):
    return DiT(depth=24, hidden_size=1024, num_heads=16, **kwargs)


DiT_models = {"DiT-S": DiT_S, "DiT-B": DiT_B, "DiT-L": DiT_L}


class ActionModel(nn.Module):
    def __init__(self, token_size, model_type, in_channels, future_action_window_size, past_action_window_size,
                 diffusion_steps=100, noise_schedule="squaredcos_cap_v2"):
        super().__init__()
        self.in_channels = in_channels
        self.noise_schedule = noise_schedule
        self.diffusion_steps = diffusion_steps
        self.diffusion = create_diffusion(timestep_respacing="", noise_schedule=noise_schedule,
                                          diffusion_steps=diffusion_steps, sigma_small=True, learn_sigma=False)
        self.ddim_diffusion = None
        self.past_action_window_size = past_action_window_size
        self.future_action_window_size = future_action_window_size
        self.net = DiT_models[model_type](token_size=token_size, in_channels=in_channels, class_dropout_prob=0.1,
                                          learn_sigma=False, future_action_window_size=future_action_window_size,
                                          past_action_window_size=past_action_window_size)

    def loss(self, x, z, noise=None, timestep=None, force_drop_ids=None):
        """action_model.py:57-73.  noise / timestep / drop ids may be injected (parity tests); otherwise drawn by torch."""
        if noise is None:
            noise = torch.randn_like(x)
        if timestep is None:
            timestep = torch.randint(0, self.diffusion.num_timesteps, (x.size(0),), device=x.device)
        x_t = self.diffusion.q_sample(x, timestep, noise)
        noise_pred = self.net(x_t, timestep, z, force_drop_ids=force_drop_ids)
        assert noise_pred.shape == noise.shape == x.shape
        from ... import ops
        return ops.mse_loss(noise_pred, noise.to(noise_pred.dtype))

    def create_ddim(self, ddim_step=10):
        self.ddim_diffusion = create_diffusion(timestep_respacing="ddim" + str(ddim_step), noise_schedule=self.noise_schedule,
                                               diffusion_steps=self.diffusion_steps, sigma_small=True, learn_sigma=False)
        return self.ddim_diffusion


class ActionModelFM(nn.Module):
    """Reference `ActionModelFM` (action_model.py:86-169): the same DiT, trained to predict the velocity u = x - noise of the
    straight path x_t = t x + (1 - t) noise, t = randint(0, T) / T with T = `diffusion_steps` = 10."""

    def __init__(self, token_size, model_type, in_channels, future_action_window_size, past_action_window_size,
                 diffusion_steps=10, noise_schedule="squaredcos_cap_v2"):
        super().__init__()
        self.in_channels = in_channels
        self.noise_schedule = noise_schedule
        self.diffusion_steps = diffusion_steps
        self.diffusion = create_diffusion(timestep_respacing="", noise_schedule=noise_schedule,
                                          diffusion_steps=diffusion_steps, sigma_small=True, learn_sigma=False)
        self.ddim_diffusion = None
        self.past_action_window_size = past_action_window_size
        self.future_action_window_size = future_action_window_size
        self.net = DiT_models[model_type](token_size=token_size, in_channels=in_channels, class_dropout_prob=0.1,
                                          learn_sigma=False, future_action_window_size=future_action_window_size,
                                          past_action_window_size=past_action_window_size)

    def loss(self, x, z, noise=None, timestep=None, force_drop_ids=None):
        """action_model.py:118-139.  `timestep` (injected by parity tests) is the INTEGER draw randint(0, T)."""
        if noise is None:
            noise = torch.randn_like(x)
        if timestep is None:
            timestep = torch.randint(0, self.diffusion.num_timesteps, (x.size(0),), device=x.device)
        t = timestep.float() / self.diffusion.num_timesteps
        tv = t.view(-1, 1, 1)
        x32, n32 = x.float(), noise.float()
        x_t = tv * x32 + (1 - tv) * n32
        ut = self.net(x_t, t, z, force_drop_ids=force_drop_ids)
        assert ut.shape == noise.shape == x.shape
        from ... import ops
        return ops.mse_loss(ut, (x32 - n32).to(ut.dtype))

    def create_ddim(self, ddim_step=10):
        """:142-169: an `FMDiffusion` over the un-respaced T = `diffusion_steps` schedule (ddim_step is not used by it)."""
        self.ddim_diffusion = FMDiffusion(betas=get_named_beta_schedule(self.noise_schedule, self.diffusion_steps))
        return self.ddim_diffusion
