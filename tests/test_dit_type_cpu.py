"""`--dit_type` DiT-S / DiT-L action heads without a GPU: the oracle against the reference goldens of the new cases, the product's
parameter layout against the reference's, and the head_dim checks of the C ABI (refused on the host, before any launch)."""
import ctypes
import json
import os
import subprocess
import sys

import pytest
import torch

from tests import synth
from tests.dit_types import DIT_SIZES, DIT_TRAIN_CFG, DIT_TYPE_CASES, build_template, oracle_forward

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
TOL = 2e-5   # the bar of test_oracle_cpu.py: fp32 vs fp32, different summation orders
DIT_TYPES = ("DiT-S", "DiT-B", "DiT-L")


def rel(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-12))


@pytest.mark.parametrize("name", list(DIT_TYPE_CASES))
def test_oracle_matches_reference_golden(name):
    cfg = DIT_TYPE_CASES[name]
    fx = json.load(open(os.path.join(GOLDEN, f"{name}.json")))
    gold = torch.load(os.path.join(GOLDEN, f"{name}.pt"))
    assert fx["cfg"]["dit_type"] == cfg["dit_type"]
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    sd = synth.synth_state_dict(build_template(cfg), cfg["weight_seed"])
    inp = synth.synth_inputs(cfg)
    with torch.no_grad():
        out = oracle_forward(sd, cfg, inp["image_primary"], inp["image_wrist"], inp["state"], inp["text_token"],
                                 action_label=inp["action_label"], mode="train", diffusion_noise=gold["diffusion_noise"],
                                 diffusion_timestep=gold["diffusion_timestep"], diffusion_drop_ids=gold["diffusion_drop_ids"])
        o2 = oracle_forward(sd, cfg, inp["image_primary"], inp["image_wrist"], inp["state"], inp["text_token"],
                                mode="test", sample_noise=gold["sample_noise"])
    assert abs(float(out["loss_action"]) - fx["loss_action"]) < 1e-4 * abs(fx["loss_action"])
    assert rel(o2["arm_pred_action"], gold["test_arm"]) < TOL
    assert rel(o2["gripper_pred_action"], gold["test_gripper"]) < TOL
    depth, _ = DIT_SIZES[cfg["dit_type"]]
    blk = "action_model.net.blocks.{}.attn.qkv.weight"
    assert blk.format(depth - 1) in sd and blk.format(depth) not in sd


@pytest.mark.parametrize("dit_type", DIT_TYPES)
def test_model_state_layout_matches_reference(dit_type):
    """The whole model of the train.main test (tests/test_dit_type_gpu.py), per dit_type: entry names and shapes as the
    reference's, recorded by tests/golden/make_golden_dit_types.py."""
    ref = {k: tuple(v) for k, v in json.load(open(os.path.join(GOLDEN, "dit_types_state.json")))[dit_type].items()}
    mine = {k: tuple(v.shape) for k, v in build_template(dict(DIT_TRAIN_CFG, dit_type=dit_type)).items()}
    assert mine == ref


_REF_DIT_SHAPES = """
import json, sys
from oracle import ref_shims
ref_shims.install()
from models.action_model.action_model import DiT_models
kw = dict(token_size=1024, in_channels=7, class_dropout_prob=0.1, learn_sigma=False, future_action_window_size=2,
          past_action_window_size=0)
print(json.dumps({t: {k: list(v.shape) for k, v in f(**kw).state_dict().items()} for t, f in DiT_models.items()}))
"""


@pytest.fixture(scope="module")
def reference_dit_shapes(repo_root):
    """Entry names and shapes of the reference's own DiT_models (action_model.py:13-21), built through oracle.ref_shims in a
    child process: the reference's top-level `models` / `utils` / `train` modules must not shadow this repository's."""
    from oracle import ref_shims
    if not ref_shims.reference_available():
        pytest.skip("reference tree not available")
    r = subprocess.run([sys.executable, "-c", _REF_DIT_SHAPES], cwd=repo_root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("dit_type", DIT_TYPES)
def test_dit_matches_reference_module(dit_type, reference_dit_shapes):
    """The product's DiT for each size against the reference's (needs the reference tree)."""
    from dreamvla_b200.models.action_model.action_model import DiT_models as MINE
    kw = dict(token_size=1024, in_channels=7, class_dropout_prob=0.1, learn_sigma=False, future_action_window_size=2,
              past_action_window_size=0)
    net = MINE[dit_type](**kw)
    ref = {k: tuple(v) for k, v in reference_dit_shapes[dit_type].items()}
    assert {k: tuple(v.shape) for k, v in net.state_dict().items()} == ref
    assert (len(net.blocks), net.num_heads) == DIT_SIZES[dit_type]
    assert ref["x_embedder.linear.weight"][0] // net.num_heads == (96 if dit_type == "DiT-S" else 64)


# ---- C ABI: head_dim is checked on the host before anything is launched -------------------------------------------------
DVLA_ERR_UNSUPPORTED = -3


def _fake_attn_args(cls, B=2, H=4, Lq=6, Lk=6, hd=96):
    """Args with 16-byte aligned pointers that are never dereferenced: every call below is refused by its host-side checks."""
    from dreamvla_b200 import _lib as L
    a = cls()
    ptr_fields = [n for n, t in cls._fields_ if t is L._vp]
    for i, n in enumerate(ptr_fields):
        setattr(a, n, 4096 * (i + 1))
    a.mask, a.tile_flags, a.key_bias = None, None, None
    if hasattr(a, "mask_t"):
        a.mask_t = None
    a.B, a.H, a.Lq, a.Lk, a.head_dim = B, H, Lq, Lk, hd
    for t in ("q", "k", "v", "o", "do", "dq", "dk", "dv"):     # [B, L, H, hd] contiguous
        if hasattr(a, f"{t}_sb"):
            L_ = Lk if t in ("k", "v", "dk", "dv") else Lq
            setattr(a, f"{t}_sb", L_ * H * hd), setattr(a, f"{t}_ss", H * hd), setattr(a, f"{t}_sh", hd)
    a.scale = hd ** -0.5
    return a


@pytest.mark.parametrize("fn", ["dvla_attn_fwd", "dvla_attn_bwd"])
@pytest.mark.parametrize("case", ["lq33", "lk65", "mask", "dropout", "hd32", "hd128", "hd128_small"])
def test_attention_rejects_unsupported_head_dim(fn, case):
    from dreamvla_b200 import _lib as L
    lib = L.load()
    cls = L.AttnFwdArgs if fn == "dvla_attn_fwd" else L.AttnBwdArgs
    kw = dict(lq33=dict(Lq=33), lk65=dict(Lk=65), hd32=dict(hd=32, Lq=100, Lk=100), hd128=dict(hd=128, Lq=100, Lk=100),
              hd128_small=dict(hd=128)).get(case, {})
    a = _fake_attn_args(cls, **kw)
    if case == "mask":
        a.mask, a.tile_flags, a.mask_words = 8192 * 16, 8192 * 17, 1
    if case == "dropout":
        a.dropout_p = 0.1
    n0 = lib.dvla_launch_count()
    rc = getattr(lib, fn)(ctypes.byref(a), None)
    msg = lib.dvla_last_error().decode()
    assert rc == DVLA_ERR_UNSUPPORTED, (case, rc, msg)
    assert "head_dim" in msg and "Lq <= 32, Lk <= 64" in msg, msg
    assert lib.dvla_launch_count() == n0


def test_attention_head_dim_zero_means_64():
    """A caller that predates the field leaves it 0: the check passes it like 64 (the call then fails on the host for
    another reason here -- a key bias outside the short-sequence case -- without launching)."""
    from dreamvla_b200 import _lib as L
    lib = L.load()
    for hd_field in (0, 64):
        a = _fake_attn_args(L.AttnFwdArgs, Lq=100, Lk=100, hd=64)
        a.head_dim = hd_field
        a.key_bias = 8192 * 16
        n0 = lib.dvla_launch_count()
        assert lib.dvla_attn_fwd(ctypes.byref(a), None) == DVLA_ERR_UNSUPPORTED
        msg = lib.dvla_last_error().decode()
        assert "key_bias" in msg and "head_dim" not in msg, msg
        assert lib.dvla_launch_count() == n0


def test_fused_sampler_rejects_head_dim_80():
    from dreamvla_b200 import _lib as L
    lib = L.load()
    depth, hidden, heads = 2, 640, 8                    # head_dim 80
    blocks = (L.DitBlockWeights * depth)(*[L.DitBlockWeights(*[4096 * (i + 1)] * 8) for i in range(depth)])
    a = L.DitSamplerArgs()
    for n, t in L.DitSamplerArgs._fields_:
        if t is L._vp:
            setattr(a, n, 8192)
    a.blocks = blocks
    a.depth, a.hidden, a.heads, a.mlp, a.token, a.freq, a.channels, a.T, a.batch = depth, hidden, heads, 4 * hidden, 1024, 256, 7, 3, 1
    a.n_steps, a.cfg_scale, a.workspace_bytes = 10, 1.5, 1 << 30
    n0 = lib.dvla_launch_count()
    rc = lib.dvla_dit_ddim_sample(ctypes.byref(a), None)
    msg = lib.dvla_last_error().decode()
    assert rc == DVLA_ERR_UNSUPPORTED and "head_dim" in msg and "hidden 640, heads 8" in msg, (rc, msg)
    assert lib.dvla_launch_count() == n0
