"""Host-side pieces of batched rollouts (no GPU): the per-timestep token layout of DreamVLA.rollout_actions against the
reference mask rules, and the argument checks of the per-sequence attention mask made before any launch."""
import ctypes

import pytest
import torch

from dreamvla_b200 import _lib, build
from dreamvla_b200.models.dreamvla_model import batched_rollout_layout, generate_attention_mask, prune_closure
from tests import synth

N_A, ACT = 36, 3


def mask_of(S, n_obs, **kw):
    args = dict(atten_goal=0, atten_goal_state=False, atten_only_obs=False, attn_robot_proprio_state=False, mask_l_obs_ratio=0.0)
    args.update(kw)
    return generate_attention_mask(K=S, num_A=N_A, num_B=n_obs + ACT, num_obs_token=n_obs, action_pred_steps=ACT, **args) == 0


def synth_n_obs(cfg):
    heads = sum(bool(cfg.get(k)) for k in ("obs_pred", "depth_pred", "dino_feat_pred", "sam_feat_pred", "trajectory_pred"))
    return 2 * cfg["num_obs_token_per_image"] * heads


CONFIGS = {
    "eval.sh": (10, 54),                  # obs + depth + SAM queries, S = 10: L_b = 417
    "libero": (7, 0),                     # world heads off, S = 7
    **{name: (cfg["sequence_length"], synth_n_obs(cfg)) for name, cfg in synth.CASES.items() if cfg["use_dit_head"]},
}


@pytest.mark.parametrize("name", list(CONFIGS))
def test_batched_layout_is_constant_prefixed_and_keeps_the_action_rows_view(name):
    S, n_obs = CONFIGS[name]
    vis = mask_of(S, n_obs)
    n_tok = N_A + n_obs + ACT
    idx, r0 = batched_rollout_layout(vis, S, N_A, ACT)
    assert idx.shape == (S, N_A * S + n_obs + ACT)
    if name == "eval.sh":
        assert idx.shape[1] == 417
    for sel in range(S):
        rows = idx[sel]
        kept = prune_closure(vis, sel, n_tok)
        assert torch.equal(rows[:len(kept)], kept)                         # the single-env sequence is a prefix
        assert bool((rows[1:] > rows[:-1]).all())                          # reference token order
        mb = vis[rows][:, rows]
        assert not bool(mb[:len(kept), len(kept):].any())                  # no kept row sees an appended slot
        a0 = sel * n_tok + n_tok - ACT
        assert torch.equal(rows[r0[sel]:r0[sel] + ACT], torch.arange(a0, a0 + ACT))
        for j in range(ACT):                                               # action rows see exactly the reference's columns
            assert torch.equal(rows[mb[r0[sel] + j]], vis[a0 + j].nonzero().flatten())


def test_batched_layout_takes_the_goal_mask_and_refuses_a_causal_one():
    S, n_obs = 5, 18
    vis = mask_of(S, n_obs, atten_goal=4, atten_goal_state=True, atten_only_obs=True, attn_robot_proprio_state=True)
    idx, _ = batched_rollout_layout(vis, S, N_A, ACT)
    for sel in range(S):
        kept = prune_closure(vis, sel, N_A + n_obs + ACT)
        assert torch.equal(idx[sel][:len(kept)], kept)
    # token-causal: timestep sel keeps every slot up to its own, so the batched length would grow with sel
    L = S * (N_A + n_obs + ACT)
    with pytest.raises(ValueError, match="kept-token count differs"):
        batched_rollout_layout(torch.ones(L, L, dtype=torch.bool).tril(), S, N_A, ACT)


@pytest.fixture(scope="module")
def lib():
    build.build_library()
    return _lib.load()


def attn_args(**kw):
    a = _lib.AttnFwdArgs()
    a.q = a.k = a.v = a.o = 1 << 20                  # never dereferenced: the checks below return before any launch
    a.B, a.H, a.Lq, a.Lk, a.head_dim = 4, 2, 128, 128, 64
    a.q_sb = a.k_sb = a.v_sb = a.o_sb = 128 * 2 * 64
    a.q_ss = a.k_ss = a.v_ss = a.o_ss = 2 * 64
    a.q_sh = a.k_sh = a.v_sh = a.o_sh = 64
    a.scale = 0.125
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_mask_index_without_mask_is_invalid(lib):
    rc = lib.dvla_attn_fwd(ctypes.byref(attn_args(mask_index=1 << 21)), None)
    assert rc == -1 and b"mask_index given without mask" in lib.dvla_last_error()


def test_negative_mask_stack_strides_are_invalid(lib):
    a = attn_args(mask=1 << 22, tile_flags=1 << 23, mask_words=4, mask_index=1 << 21, mask_stride=-512, flags_stride=4)
    rc = lib.dvla_attn_fwd(ctypes.byref(a), None)
    assert rc == -1 and b"negative mask_stride" in lib.dvla_last_error()

