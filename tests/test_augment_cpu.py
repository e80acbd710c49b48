"""oracle/augment_oracle.py against the reference's own `RandomShiftsAug` / `depth_image_fn` (tests/golden/augment.pt, produced
by tests/golden/make_golden_augment.py from the unmodified reference code, and the digest of one reference trajectory in
tests/golden/reference_checks.pt),
and the closed form the CUDA kernel implements (a clamped crop) against the reference's grid_sample formulation."""
import os

import pytest
import torch

from oracle import augment_oracle as ao

GOLD = os.path.join(os.path.dirname(__file__), "golden", "augment.pt")


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD)


@pytest.mark.parametrize("name", ["rgb", "gripper", "depth"])
def test_grid_sample_restatement_matches_reference(gold, name):
    g = gold[name]
    x, pad = g["x"], g["pad"]
    n, t = x.shape[:2]
    y = ao.random_shifts_grid_sample_traj(x, g["traj_shifts"], pad)
    assert torch.equal(y, g["traj"]), "forward_traj restatement differs from the reference output"
    y = ao.random_shifts_grid_sample(x.view(n * t, *x.shape[2:]), g["fwd_shifts"], pad)
    assert torch.equal(y, g["fwd"]), "forward restatement differs from the reference output"
    assert int(g["traj_shifts"].min()) >= 1 and int(g["traj_shifts"].max()) <= 2 * pad and int(g["fwd_shifts"].min()) >= 0


@pytest.mark.parametrize("name", ["rgb", "gripper", "depth"])
def test_clamped_crop_equals_the_reference_up_to_grid_rounding(gold, name):
    """What dvla_shift_crop computes vs the reference: the fp32 grid coordinates miss the pixel centres by ~1e-5 pixels, so the
    reference's bilinear sample mixes in at most that fraction of a neighbouring pixel."""
    g = gold[name]
    x, pad = g["x"], g["pad"]
    n, t = x.shape[:2]
    crop = ao.shift_crop(x.view(n * t, *x.shape[2:]), g["traj_shifts"], pad).view_as(x)
    scale = float(x.abs().max())
    assert float((crop - g["traj"]).abs().max()) <= 2e-4 * scale
    crop = ao.shift_crop(x.view(n * t, *x.shape[2:]), g["fwd_shifts"], pad)
    assert float((crop - g["fwd"]).abs().max()) <= 2e-4 * scale
    # and it is a pure gather: every output value is an input value of the same image / channel
    assert torch.isin(crop[0, 0], x.view(n * t, *x.shape[2:])[0, 0]).all()


def test_draw_matches_reference_stream():
    torch.manual_seed(11)
    a = ao.draw_shifts(6, 10, 1)
    torch.manual_seed(11)
    b = torch.randint(1, 21, size=(6, 1, 1, 2), dtype=torch.float32).view(6, 2).to(torch.int32)
    assert torch.equal(a, b)


def test_nearest_resize_matches_reference(gold):
    ys, xs = gold["resize_rows_200_to_224"].long(), gold["resize_cols_200_to_224"].long()
    coord = torch.arange(200 * 200, dtype=torch.float32).view(1, 200, 200)
    mine = ao.resize_nearest(coord, 224, 224)[0].long()
    assert torch.equal(mine, ys.view(-1, 1) * 200 + xs.view(1, -1)), "200 -> 224 index map differs from torchvision NEAREST"
    small = ao.resize_nearest(gold["resize_small_in"], 224, 224).unsqueeze(1)
    assert torch.equal(small.to(torch.float16), gold["resize_small_out"])


def test_live_reference_code(gold):
    """RandomShiftsAug.forward_traj of the reference on a seeded batch (its output's digest recorded by
    tests/golden/make_golden_reference_checks.py) vs the oracle's grid_sample restatement and clamped crop."""
    from tests.digests import digest
    ref = torch.load(os.path.join(os.path.dirname(__file__), "golden", "reference_checks.pt"))["augment_traj"]
    pad = gold["rgb"]["pad"]
    x = torch.randn(3, 2, 3, 56, 56, generator=torch.Generator().manual_seed(ref["x_seed"]))
    torch.manual_seed(ref["torch_seed"])
    s = ao.draw_shifts(6, pad, 1)
    mine = ao.random_shifts_grid_sample_traj(x, s, pad)
    assert digest(mine) == ref["traj"], "grid_sample restatement differs from the reference's RandomShiftsAug"
    assert float((ao.shift_crop(x.view(6, 3, 56, 56), s, pad).view_as(x) - mine).abs().max()) <= 2e-4 * float(x.abs().max())
