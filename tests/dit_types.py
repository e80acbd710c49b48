"""Action-head sizes (`--dit_type`, reference models/action_model/action_model.py:13-21) in the test infrastructure.

The shared fixtures (tests/synth.py, oracle/dreamvla_oracle.py) describe the default DiT-B head; this module adds the other
two sizes on top of them without changing what they compute:
  * DIT_TYPE_CASES / DIT_TRAIN_CFG: synthetic configurations with a `dit_type`, and `ctor_kwargs` that passes it on;
  * `oracle_forward`: oracle.dreamvla_forward with the DiT depth and head count of the configuration's `dit_type`;
  * `build_template`: the product model's state_dict (names, shapes, fixed buffers) for such a configuration, on the CPU.
Used by tests/test_dit_type_{cpu,gpu}.py and tests/golden/make_golden_dit_types.py.
"""
from __future__ import annotations

import contextlib
import functools

import torch

from tests import synth

# action_model.py:13-21: (depth, heads) of each size; the hidden width is read from the weights
DIT_SIZES = {"DiT-S": (6, 4), "DiT-B": (12, 12), "DiT-L": (24, 16)}

# reference -> golden -> oracle on the CPU, CUDA path on the GPU; each with its own seeds.  DiT-S has head_dim 96.
DIT_TYPE_CASES = {
    "libero_dit_s": dict(synth.CASES["libero_dit"], dit_type="DiT-S", weight_seed=51, input_seed=52, draw_seed=53),
    "libero_dit_l": dict(synth.CASES["libero_dit"], dit_type="DiT-L", weight_seed=61, input_seed=62, draw_seed=63),
    "libero_fm_dit_s": dict(synth.FM_CASES["libero_fm"], dit_type="DiT-S", weight_seed=71, input_seed=72, draw_seed=73),
}

# The model tests/test_dit_type_gpu.py trains through train.main (its command-line flags), one per `dit_type`; the
# reference's state_dict layout of it is recorded in tests/golden/dit_types_state.json.
DIT_TRAIN_CFG = dict(synth.BASE, obs_pred=True, depth_pred=False, trajectory_pred=False, dino_feat_pred=False,
                     sam_feat_pred=False, use_dit_head=True)


def ctor_kwargs(cfg):
    """synth.ctor_kwargs plus the action-head size."""
    kw = synth.ctor_kwargs(cfg)
    if "dit_type" in cfg:
        kw["dit_type"] = cfg["dit_type"]
    return kw


@contextlib.contextmanager
def _dit_size(O, dit_type):
    # dreamvla_forward calls the module-level dit_forward with its DiT-B defaults (depth 12, heads 12)
    depth, heads = DIT_SIZES[dit_type]
    orig = O.dit_forward
    O.dit_forward = functools.partial(orig, depth=depth, heads=heads)
    try:
        yield
    finally:
        O.dit_forward = orig


def oracle_forward(sd, cfg, *args, **kwargs):
    """oracle.dreamvla_forward for a configuration of any `dit_type` (default DiT-B)."""
    from oracle import dreamvla_oracle as O
    with _dit_size(O, cfg.get("dit_type", "DiT-B")):
        return O.dreamvla_forward(sd, cfg, *args, **kwargs)


@functools.lru_cache(maxsize=4)
def _template(cfg_items):
    from dreamvla_b200.models import DreamVLA
    torch.manual_seed(0)
    m = DreamVLA(finetune_type="calvin", clip_device="cpu", vit_checkpoint_path=None, **ctor_kwargs(dict(cfg_items)))
    return {k: v.detach().clone() for k, v in m.state_dict().items()}


def build_template(cfg):
    """tests/state_template.build_template for a configuration with a `dit_type`."""
    return _template(tuple(sorted(cfg.items())))
