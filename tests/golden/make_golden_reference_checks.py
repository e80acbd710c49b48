"""Generates tests/golden/reference_checks.pt FROM THE UNMODIFIED REFERENCE (DreamVLA tree + oracle/ref_shims.py): the
reference-side values that tests/test_mask_cpu.py, tests/test_oracle_cpu.py and tests/test_augment_cpu.py compare the
product and the oracle against, so that those comparisons run without the reference tree.

    DVLA_REFERENCE_ROOT=<DreamVLA checkout> python tests/golden/make_golden_reference_checks.py

Tensors compared bit for bit are stored as the SHA-256 of their bytes, large tensors as a fixed strided sample of their
elements plus their float64 sum (tests/digests.py).  Both keep the file small.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from oracle import ref_shims  # noqa: E402
from tests import synth  # noqa: E402
from tests.digests import digest, sample  # noqa: E402

def mask_checks():
    from tests.test_mask_cpu import COMBOS
    ref_shims.install()
    from models.dreamvla_model import generate_attention_mask as gen_ref
    out = []
    for kw in COMBOS[::7]:
        np.random.seed(5)
        m = gen_ref(**kw)
        out.append({"kw": kw, "digest": digest(m)})
    return out


def state_keys():
    import make_golden
    model = make_golden.build_reference(synth.CASES["calvin_allheads"])
    ref = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    return {k: v for k, v in ref.items() if not (k.startswith("vision_encoder.decoder") or k == "vision_encoder.mask_token")}


def loss_helpers():
    ref_shims.install()
    from utils import train_utils as R
    from utils.sigloss import SiLogLoss
    g = torch.Generator().manual_seed(3)
    imgs = torch.randn(3, 3, 224, 224, generator=g)
    x = R.patchify(imgs, 16)
    pt = torch.rand(2, 1, 196, 256, generator=g) + 0.1
    tgt = torch.rand(2, 1, 1, 224, 224, generator=g) * 4 + 0.1
    return {"patchify": sample(x), "normalize": sample(R.normalize_patchfied_image(x)), "unpatchify": sample(R.unpatchify(pt)),
            "silog": float(SiLogLoss()(R.unpatchify(pt), tgt))}


def augment_traj():
    from make_golden_augment import reference_namespace
    gold = torch.load(os.path.join(HERE, "augment.pt"))
    pad = gold["rgb"]["pad"]
    aug = reference_namespace()["RandomShiftsAug"](pad)
    x = torch.randn(3, 2, 3, 56, 56, generator=torch.Generator().manual_seed(21))
    torch.manual_seed(5)
    return {"x_seed": 21, "torch_seed": 5, "traj": digest(aug.forward_traj(x.clone()))}


if __name__ == "__main__":
    torch.save({"mask": mask_checks(), "state_keys": state_keys(), "loss_helpers": loss_helpers(), "augment_traj": augment_traj()},
               os.path.join(HERE, "reference_checks.pt"))
    print("wrote", os.path.join(HERE, "reference_checks.pt"))
