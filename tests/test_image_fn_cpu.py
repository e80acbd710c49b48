"""CLIP's image transform (`image_processor`) without a GPU: the library's host-side Pillow coefficients (dvla_bicubic_coeffs),
run through a numpy restatement of Pillow's two integer passes, reproduce the torchvision + Pillow crops bit for bit
(tests/golden/image_fn.pt, and live Pillow when it is installed); the Normalize table equals ToTensor + Normalize on every
uint8 value; and the train loop's host logic (`data_utils.prepare_batch`) preprocesses raw uint8 windows before the random
shifts, with the C-ABI calls replaced by closed forms."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from dreamvla_b200 import _lib as L
from dreamvla_b200.utils import data_utils as du
from oracle import augment_oracle as ao

_spec = importlib.util.spec_from_file_location(
    "make_golden_image_fn", os.path.join(os.path.dirname(__file__), "golden", "make_golden_image_fn.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)


@pytest.fixture(scope="module")
def lib():
    from dreamvla_b200 import build
    build.build_library()
    return L.load()


def clip8(v):
    return np.where(v <= 0, 0, np.where(v >= 1 << 30, 255, v >> 22)).astype(np.uint8)


def resample_line(x, bounds, coeffs, axis):
    """Pillow's 8-bit pass along `axis` of x (uint8 [..., n, ..., 3]) with the given bounds / int32 coefficients."""
    n = x.shape[axis]
    taps = coeffs.shape[1]
    idx = np.minimum(bounds[:, :1] + np.arange(taps)[None, :], n - 1)                  # [count, taps]; coefficient 0 past the taps
    g = np.take(x.astype(np.int64), idx, axis=axis)                                     # axis -> (count, taps)
    shape = [1] * g.ndim
    shape[axis], shape[axis + 1] = coeffs.shape
    s = (1 << 21) + (g * coeffs.astype(np.int64).reshape(shape)).sum(axis=axis + 1)
    return clip8(s)


def crop_numpy(frame, flip=False):
    """uint8 [h, w, 3] -> uint8 [224, 224, 3]: the library's coefficients, Pillow's passes (horizontal, then vertical)."""
    f = np.asarray(frame)[::-1] if flip else np.asarray(frame)
    h, w = f.shape[:2]
    rh, rw, top, left = L.image_fn_geometry(h, w)
    xb, xc = (t.numpy() for t in L.bicubic_coeffs(w, rw, left, 224))
    yb, yc = (t.numpy() for t in L.bicubic_coeffs(h, rh, top, 224))
    return resample_line(resample_line(f, xb, xc, axis=1), yb, yc, axis=0)


def test_geometry_matches_torchvision():
    from torchvision.transforms.functional import _compute_resized_output_size
    for h, w in G.SHAPES + [(203, 200), (200, 203), (225, 3584), (1, 1), (3584, 224)]:
        rh, rw, top, left = L.image_fn_geometry(h, w)
        assert [rh, rw] == _compute_resized_output_size((h, w), [224]), (h, w)
        assert (top, left) == (int(round((rh - 224) / 2.0)), int(round((rw - 224) / 2.0)))
    assert L.image_fn_geometry(203, 200) == (227, 224, 2, 0), "Python's round: 1.5 -> 2"
    assert L.image_fn_geometry(7, 5)[2] == 44, "Python's round: 44.5 -> 44"


def test_coefficients_reproduce_golden_crops(lib):
    crops, gold = G.load_crops()
    assert len(crops) == 2 * len(G.SHAPES)
    for name, frame in G.make_inputs(gold["seed"], gold["shapes"]):
        got = crop_numpy(frame.numpy())
        want = crops[name].numpy()
        assert np.array_equal(got, want), (name, int((got != want).sum()))


def test_coefficients_match_live_pillow(lib):
    pytest.importorskip("PIL")
    pytest.importorskip("torchvision")
    shapes = [(200, 200), (84, 84), (128, 128), (203, 200), (200, 203), (257, 511), (97, 1500), (224, 300)]
    for seed in (1, 2):
        for name, frame in G.make_inputs(seed, shapes):
            want = G.clip_crop(frame).numpy()
            assert np.array_equal(crop_numpy(frame.numpy()), want), (seed, name)
            flipped = G.clip_crop(frame.flip(0)).numpy()
            assert np.array_equal(crop_numpy(frame.numpy(), flip=True), flipped), (seed, name, "flip")


def test_coefficient_tables(lib):
    b, c = L.bicubic_coeffs(224, 224, 0, 224)
    assert c.shape == (224, 1) and torch.equal(b[:, 0], torch.arange(224, dtype=torch.int32)) and bool((b[:, 1] == 1).all())
    assert bool((c == 1 << 22).all()), "an unchanged size is the identity"
    assert int(lib.dvla_bicubic_taps(200, 224)) == 5 and int(lib.dvla_bicubic_taps(1000, 224)) == 19
    b, c = L.bicubic_coeffs(1000, 224, 0, 224)
    assert c.shape == (224, 19)
    sums = c.sum(1)
    assert int((sums - (1 << 22)).abs().max()) <= 19, "normalised by their sum, rounded per tap"
    for i in range(224):
        assert bool((c[i, int(b[i, 1]):] == 0).all())
    assert int(lib.dvla_bicubic_taps(0, 224)) < 0
    bounds, coeffs = torch.zeros(2, 2, dtype=torch.int32), torch.zeros(2, 5, dtype=torch.int32)
    assert lib.dvla_bicubic_coeffs(200, 224, 223, 2, bounds.data_ptr(), coeffs.data_ptr()) == -1, "outputs past out_size"
    assert b"out of range" in lib.dvla_last_error()


def test_lut_is_totensor_normalize():
    T = pytest.importorskip("torchvision.transforms")
    from PIL import Image
    v = np.repeat(np.arange(256, dtype=np.uint8)[None, :, None], 3, axis=2)            # [1, 256, 3]: every value, every channel
    want = T.Normalize(du.CLIP_MEAN, du.CLIP_STD)(T.ToTensor()(Image.fromarray(v)))[:, 0, :]
    assert torch.equal(du.image_fn_lut("cpu"), want)


# ---- train-loop host logic --------------------------------------------------------------------------------------------------
def fake_image_fn(calls):
    def f(frames, lut, out_dtype=torch.float32, flip_vertical=False):
        calls.append(("image_fn", tuple(frames.shape), out_dtype))
        crops = np.stack([crop_numpy(fr, flip_vertical) for fr in frames.numpy()])          # [n, 224, 224, 3]
        idx = torch.from_numpy(crops).long().permute(0, 3, 1, 2)                            # [n, 3, 224, 224]
        return torch.stack([lut[c][idx[:, c]] for c in range(3)], dim=1).to(out_dtype)
    return f


def fake_shift_crop(calls):
    def f(x, shifts, pad, out_dtype=None):
        calls.append(("shift_crop", tuple(x.shape), shifts.clone(), pad))
        return ao.shift_crop(x.float(), shifts, pad).to(out_dtype or x.dtype)
    return f


def raw_batch():
    g = torch.Generator().manual_seed(4)
    return {"images_primary": torch.randint(0, 256, (1, 2, 20, 24, 3), generator=g, dtype=torch.uint8),
            "images_wrist": torch.randint(0, 256, (1, 2, 12, 12, 3), generator=g, dtype=torch.uint8),
            "states": torch.zeros(1, 2, 15), "text": torch.zeros(1, 77, dtype=torch.long)}


def test_raw_frames_are_preprocessed_before_the_shifts(lib, monkeypatch):
    calls = []
    monkeypatch.setattr(L, "image_fn", fake_image_fn(calls))
    monkeypatch.setattr(L, "shift_crop", fake_shift_crop(calls))
    b = raw_batch()
    out = du.prepare_batch(b, rgb_pad=10, gripper_pad=4, traj_cons=True, device_augment=True, generator=torch.Generator().manual_seed(1))
    assert [c[0] for c in calls] == ["image_fn", "image_fn", "shift_crop", "shift_crop"]
    assert calls[0][1:] == ((2, 20, 24, 3), torch.bfloat16) and calls[1][1:] == ((2, 12, 12, 3), torch.bfloat16)
    assert [c[1] for c in calls[2:]] == [(2, 3, 224, 224), (2, 3, 224, 224)] and [c[3] for c in calls[2:]] == [10, 4]
    lut = du.image_fn_lut("cpu")
    pre = fake_image_fn([])(b["images_primary"].view(2, 20, 24, 3), lut, torch.bfloat16)
    want = ao.shift_crop(pre.float(), calls[2][2], 10).to(torch.bfloat16).view(1, 2, 3, 224, 224)
    assert out["images_primary"].dtype == torch.bfloat16 and torch.equal(out["images_primary"], want)
    assert out["states"] is b["states"] and b["images_primary"].dtype == torch.uint8, "the input batch is not modified"


def test_raw_frames_without_shifts(lib, monkeypatch):
    calls = []
    monkeypatch.setattr(L, "image_fn", fake_image_fn(calls))
    monkeypatch.setattr(L, "shift_crop", fake_shift_crop(calls))
    out = du.prepare_batch(raw_batch(), rgb_pad=-1, gripper_pad=-1, device_augment=False)
    assert [c[0] for c in calls] == ["image_fn", "image_fn"]
    assert out["images_wrist"].shape == (1, 2, 3, 224, 224) and out["images_wrist"].dtype == torch.bfloat16


def test_raw_frames_with_pads_need_device_augment(monkeypatch):
    calls = []
    monkeypatch.setattr(L, "image_fn", fake_image_fn(calls))
    with pytest.raises(ValueError, match="--device_augment"):
        du.prepare_batch(raw_batch(), rgb_pad=10, gripper_pad=-1, device_augment=False)
    assert not calls


def test_float_batches_are_untouched(monkeypatch):
    calls = []
    monkeypatch.setattr(L, "image_fn", fake_image_fn(calls))
    monkeypatch.setattr(L, "shift_crop", fake_shift_crop(calls))
    b = {"images_primary": torch.randn(1, 2, 3, 16, 16), "images_wrist": torch.randn(1, 2, 3, 16, 16)}
    assert du.prepare_batch(b, rgb_pad=10, gripper_pad=4, device_augment=False) is b
    assert du.prepare_batch(b, rgb_pad=-1, gripper_pad=-1, device_augment=True) is b
    out = du.prepare_batch(b, rgb_pad=2, gripper_pad=-1, device_augment=True, generator=torch.Generator().manual_seed(3))
    assert [c[0] for c in calls] == ["shift_crop"] and out["images_wrist"] is b["images_wrist"]
