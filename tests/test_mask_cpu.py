"""Bit-exact contract for the attention mask (dreamvla_model.py:25-66): product generator == oracle generator ==
reference generator (its masks' digests in tests/golden/reference_checks.pt) == golden packed mask, for every flag combination the shipped scripts use."""
import itertools
import json
import os

import numpy as np
import pytest
import torch

from dreamvla_b200.models.dreamvla_model import generate_attention_mask as gen_product
from dreamvla_b200.ops import AttnMask
from oracle.dreamvla_oracle import generate_attention_mask as gen_oracle
from tests import synth
from tests.digests import digest

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
COMBOS = [dict(K=K, num_A=36, num_B=nobs + 3, atten_goal=ag, atten_goal_state=ags, atten_only_obs=aoo,
               attn_robot_proprio_state=arp, mask_l_obs_ratio=r, num_obs_token=nobs, action_pred_steps=3)
          for K, nobs, (ag, ags), aoo, arp, r in itertools.product(
              (2, 7, 10), (0, 18, 90), ((0, False), (4, True), (2, False)), (False, True), (False, True), (0.0, 0.5))]


@pytest.mark.parametrize("kw", COMBOS[::5])
def test_product_equals_oracle(kw):
    np.random.seed(3)
    a = gen_product(**kw)
    np.random.seed(3)
    b = gen_oracle(**kw)
    assert torch.equal(a, b)


@pytest.mark.parametrize("kw", COMBOS[::7])
def test_product_equals_reference(kw):
    np.random.seed(5)
    a = gen_product(**kw)
    ref = torch.load(os.path.join(GOLDEN, "reference_checks.pt"))["mask"][COMBOS[::7].index(kw)]
    assert ref["kw"] == kw
    assert digest(a) == ref["digest"], "mask differs from the reference generator's"


@pytest.mark.parametrize("name", list(synth.CASES))
def test_matches_golden_packed_mask(name):
    cfg = synth.CASES[name]
    gold = torch.load(os.path.join(GOLDEN, f"{name}.pt"))
    fx = json.load(open(os.path.join(GOLDEN, f"{name}.json")))
    n_obs = 18 * sum(bool(cfg.get(k)) for k in ("obs_pred", "depth_pred", "dino_feat_pred", "sam_feat_pred", "trajectory_pred"))
    m = gen_product(K=cfg["sequence_length"], num_A=36, num_B=n_obs + 3, atten_goal=cfg.get("atten_goal", False),
                    atten_goal_state=cfg.get("atten_goal_state", False), atten_only_obs=cfg.get("atten_only_obs", False),
                    attn_robot_proprio_state=cfg.get("attn_robot_proprio_state", False),
                    mask_l_obs_ratio=cfg.get("mask_l_obs_ratio", 0.0), num_obs_token=n_obs, action_pred_steps=3)
    vis = (m == 0)
    assert list(vis.shape) == fx["mask_shape"] and int(vis.sum()) == fx["mask_visible_pairs"]
    assert torch.equal(torch.from_numpy(np.packbits(vis.numpy(), axis=1)), gold["mask_packed"])


def test_bit_packing_roundtrip():
    g = torch.Generator().manual_seed(0)
    vis = torch.rand(70, 131, generator=g) < 0.4
    bits = AttnMask.pack_bits(vis)
    assert bits.shape == (70, 5) and bits.dtype == torch.int32
    words = bits.to(torch.int64) & 0xFFFFFFFF
    back = ((words.unsqueeze(-1) >> torch.arange(32)) & 1).bool().reshape(70, -1)[:, :131]
    assert torch.equal(back, vis)
    assert not ((words.unsqueeze(-1) >> torch.arange(32)) & 1).bool().reshape(70, -1)[:, 131:].any()

