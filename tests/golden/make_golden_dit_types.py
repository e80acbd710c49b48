"""Generates the `--dit_type` fixtures under tests/golden/ FROM THE UNMODIFIED REFERENCE (DreamVLA tree + oracle/ref_shims.py):

  * <case>.pt / <case>.json for each case of tests/dit_types.DIT_TYPE_CASES (libero_dit_s, libero_dit_l, libero_fm_dit_s),
    exactly as tests/golden/make_golden.py writes its cases (run_case), with the action-head size passed to the reference;
  * dit_types_state.json: the reference model's state_dict entry names and shapes for each size (action_model.py:13-21), so
    that the product's parameter layout for DiT-S / DiT-B / DiT-L (what a checkpoint saved by train.py holds) is checked
    without the reference tree.  The model is the one tests/test_dit_type_gpu.py trains through train.main (DIT_TRAIN_CFG);
    the dead MAE decoder of the vision encoder is left out, as in tests/golden/reference_checks.pt.

    DVLA_REFERENCE_ROOT=<DreamVLA checkout> python tests/golden/make_golden_dit_types.py [case or "state" ...]
"""
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import make_golden  # noqa: E402
from oracle import ref_shims  # noqa: E402
from tests.dit_types import DIT_SIZES, DIT_TRAIN_CFG, DIT_TYPE_CASES, ctor_kwargs  # noqa: E402


def build_reference(cfg):
    """make_golden.build_reference with the action-head size passed to the reference's constructor."""
    ref_shims.install()
    from models.dreamvla_model import DreamVLA  # the reference's own class
    fake = "/tmp/_dvla_fake_vit.pth"
    if not os.path.exists(fake):
        torch.save({"model": {}}, fake)
    torch.manual_seed(0)
    model = DreamVLA(finetune_type="calvin", clip_device="cpu", vit_checkpoint_path=fake, **ctor_kwargs(cfg))
    model._init_model_type()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    return model


def state_shapes(dit_type):
    model = build_reference(dict(DIT_TRAIN_CFG, dit_type=dit_type))
    return {k: list(v.shape) for k, v in model.state_dict().items()
            if not (k.startswith("vision_encoder.decoder") or k == "vision_encoder.mask_token")}


if __name__ == "__main__":
    torch.set_num_threads(8)
    only = sys.argv[1:]
    make_golden.build_reference = build_reference          # run_case builds its reference model through this name
    for name, cfg in DIT_TYPE_CASES.items():
        if not only or name in only:
            make_golden.run_case(name, cfg)
    if not only or "state" in only:
        out = {t: state_shapes(t) for t in DIT_SIZES}
        with open(os.path.join(HERE, "dit_types_state.json"), "w") as f:
            json.dump(out, f, indent=0, sort_keys=True)
        print({t: len(v) for t, v in out.items()})
