"""Host restatement of the pretrain phase's device-drawn observation-token drop (include/dvla.h dvla_attn_mask_obs_drop) and
what it must satisfy without a GPU: `count` distinct columns per timestep, uniform single-column and column-pair drop
frequencies, independent timesteps, and -- given the same subsets -- the reference's mask (dreamvla_model.py:25-66) bit for
bit.  tests/test_obs_drop_mask_gpu.py holds the kernel to this restatement."""
import ctypes

import numpy as np
import pytest
import torch

from dreamvla_b200.models.dreamvla_model import generate_attention_mask
from tests.philox_ref import _C2, _C3, philox4x32
from tests.test_mask_cpu import COMBOS

_LO = np.uint64(0xFFFFFFFF)


def drop_keys(seed, counter, K, n_obs):
    """uint64 [K, n_obs]: r(i, j) = philox4x32(seed + counter, i * n_obs + j).x."""
    eff = (int(seed) + int(counter)) & ((1 << 64) - 1)
    off = np.arange(K * n_obs, dtype=np.uint64)
    x = philox4x32((off & _LO, off >> np.uint64(32), _C2, _C3), (eff & 0xFFFFFFFF, eff >> 32))[0]
    return x.reshape(K, n_obs)


def dropped_columns(seed, counter, K, n_obs, count):
    """Per timestep, the `count` observation columns with the smallest (r(i, j), j), in that order."""
    r = drop_keys(seed, counter, K, n_obs)
    j = np.arange(n_obs)
    return [[int(c) for c in np.lexsort((j, r[i]))[:count]] for i in range(K)]


def restated_mask(kw, seed, counter):
    """(additive mask with mask_l_obs_ratio = 0, the same mask with the restated drop, the dropped columns)."""
    K, num_A, n_obs, n_act = kw["K"], kw["num_A"], kw["num_obs_token"], kw["action_pred_steps"]
    base = generate_attention_mask(**{**kw, "mask_l_obs_ratio": 0.0})
    drops = dropped_columns(seed, counter, K, n_obs, int(kw["mask_l_obs_ratio"] * n_obs))
    m = base.clone()
    n_tok = num_A + kw["num_B"]
    for i, cols in enumerate(drops):
        a0 = i * n_tok + num_A + n_obs
        for j in cols:
            m[a0:a0 + n_act, i * n_tok + num_A + j] = -float("inf")
    return base, m, drops


@pytest.mark.parametrize("K,n_obs,count", [(11, 18, 9), (3, 90, 45), (2, 18, 0), (2, 18, 18), (4, 7, 3)])
def test_each_timestep_drops_count_distinct_columns(K, n_obs, count):
    for seed, counter in ((0, 0), (0x243F6A8885A308D3, 1), ((1 << 64) - 1, 5)):
        for cols in dropped_columns(seed, counter, K, n_obs, count):
            assert len(cols) == len(set(cols)) == count and all(0 <= c < n_obs for c in cols)


def test_drop_frequencies_are_uniform_and_timesteps_independent():
    """Over 4000 counters: every column is dropped with probability count/n_obs, every pair of columns of one timestep with
    count(count-1)/(n_obs(n_obs-1)), and a column of timestep 0 together with one of timestep 1 with (count/n_obs)^2."""
    K, n_obs, count, N = 2, 18, 9, 4000
    hit = np.zeros((N, K, n_obs), dtype=bool)
    for c in range(N):
        for i, cols in enumerate(dropped_columns(0x9E3779B97F4A7C15, c, K, n_obs, count)):
            hit[c, i, cols] = True
    h = hit.astype(np.float64)

    def within(freq, p, n):
        sigma = np.sqrt(p * (1 - p) / n)
        worst = float(np.abs(freq - p).max() / sigma)
        assert worst < 5.0, (worst, p)

    within(h.reshape(N * K, n_obs).mean(0), count / n_obs, N * K)
    pair = np.einsum("nij,nik->jk", h, h) / (N * K)
    iu = np.triu_indices(n_obs, 1)
    within(pair[iu], count * (count - 1) / (n_obs * (n_obs - 1)), N * K)
    cross = np.einsum("nj,nk->jk", h[:, 0], h[:, 1]) / N
    within(cross.ravel(), (count / n_obs) ** 2, N)


PRETRAIN_SH = dict(K=11, num_A=36, num_B=18 + 3, atten_goal=4, atten_goal_state=True, atten_only_obs=True,
                   attn_robot_proprio_state=True, mask_l_obs_ratio=0.5, num_obs_token=18, action_pred_steps=3)
ALL_HEADS = dict(PRETRAIN_SH, K=3, num_B=90 + 3, num_obs_token=90)
DRAWN = [kw for kw in COMBOS if kw["atten_only_obs"] and kw["mask_l_obs_ratio"] > 0]


@pytest.mark.parametrize("kw", [PRETRAIN_SH, ALL_HEADS] + DRAWN)
def test_restated_drop_is_the_reference_mask_with_those_subsets(kw, monkeypatch):
    """generate_attention_mask with np.random.choice returning the restated subsets in call order == the mask without the
    drop with those (action row, observation column) pairs hidden, bit for bit."""
    for seed, counter in ((7, 0), (0xD1342543DE82EF95, 3)):
        base, want, drops = restated_mask(kw, seed, counter)
        calls = []

        def choice(a, size, replace):
            assert list(a) == list(range(kw["num_obs_token"])) and size == int(kw["mask_l_obs_ratio"] * kw["num_obs_token"])
            assert replace is False
            calls.append(drops[len(calls)])
            return np.asarray(calls[-1], dtype=np.int64)

        monkeypatch.setattr(np.random, "choice", choice)
        got = generate_attention_mask(**kw)
        assert len(calls) == (kw["K"] if kw["num_obs_token"] > 0 else 0)
        assert torch.equal(got, want)
        if kw["num_obs_token"] > 0:
            assert not torch.equal(got, base)


def test_kernel_entry_rejects_bad_arguments():
    """Argument errors are reported before anything touches the device (no GPU needed): DVLA_ERR_INVALID and a message."""
    from dreamvla_b200 import _lib
    lib = _lib.load()
    p = ctypes.c_void_p(256)       # never dereferenced: every call below fails its argument checks first

    def call(L=627, W=20, K=11, n_tok=57, num_A=36, n_obs=18, n_act=3, count=9, base=p, bits=ctypes.c_void_p(512)):
        rc = lib.dvla_attn_mask_obs_drop(base, bits, p, W, L, K, n_tok, num_A, n_obs, n_act, count, 1, None, None)
        return rc, lib.dvla_last_error().decode()

    for kw, text in ((dict(count=19), "count"), (dict(count=-1), "count"), (dict(n_obs=300, n_tok=339, L=3729, W=117), "limit"),
                     (dict(K=12), "layout"), (dict(n_tok=56, L=616), "outside"), (dict(W=19), "mask_words"),
                     (dict(bits=p), "alias"), (dict(base=None), "null"), (dict(n_obs=0), "n_obs")):
        rc, msg = call(**kw)
        assert rc == -1 and text in msg, (kw, rc, msg)
