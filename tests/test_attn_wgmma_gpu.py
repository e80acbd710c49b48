"""The TMA + wgmma attention kernels (attn_fwd_wgmma_kernel, attn_bwd_wgmma_kernel) against fp32 torch under the dropout
mask of tests/philox_ref.py, at the shapes the CALVIN train step runs them at and at the edge shapes of their tiling:
Lq = 96, Lq != Lk, sequence tails, skipped / partial / full mask tiles, a per-sequence mask stack and dropout on and off.
Every case also runs twice and must give the same bits: the backward accumulates in a fixed order, with no atomics."""
import pytest
import torch

from tests import philox_ref as R

pytestmark = pytest.mark.gpu

SCALE = 0.125
SEED = 0x5EED0FA77E57


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def L(dev):
    from dreamvla_b200 import _lib
    _lib.load()
    return _lib


def _backbone_vis():
    from dreamvla_b200.models.dreamvla_model import generate_attention_mask
    add = generate_attention_mask(K=10, num_A=36, num_B=93, atten_goal=0, atten_goal_state=False, atten_only_obs=False,
                                  attn_robot_proprio_state=False, mask_l_obs_ratio=0.0, num_obs_token=90, action_pred_steps=3)
    return add == 0


def _random_vis(Lq, Lk, g):
    """~30 % visible, key 0 always; keys 64..127 hidden from the first half of the queries (skipped tiles) and visible to
    the second half (full tiles where the half is tile aligned)."""
    m = torch.rand(Lq, Lk, generator=g) < 0.3
    m[:, 0] = True
    m[: Lq // 2, 64:128] = False
    m[Lq // 2:, 64:128] = True
    return m


# (id, B, H, Lq, Lk, mask, p, backward): mask None, "backbone" (the GPT-2 block mask of the C2 step) or "random"
CASES = [
    ("backbone_8x16x1290_p0.1", 8, 16, 1290, 1290, "backbone", 0.1, True),
    ("backbone_2x16x1290_p0", 2, 16, 1290, 1290, "backbone", 0.0, True),
    ("decoder_160x16x265", 160, 16, 265, 265, None, 0.0, True),
    ("vit_160x12x197", 160, 12, 197, 197, None, 0.0, False),
    ("lq96_p0.1", 2, 3, 96, 96, None, 0.1, True),
    ("lq96_lk200_random_p0.1", 2, 2, 96, 200, "random", 0.1, True),
    ("lq330_lk140_random_p0.1", 2, 2, 330, 140, "random", 0.1, True),
    ("lq256_lk320_random_p0", 1, 3, 256, 320, "random", 0.0, True),
    ("lq200_lk517_p0.3", 2, 2, 200, 517, None, 0.3, True),
]


def _inputs(B, H, Lq, Lk, dev, g):
    q, k, v = (torch.randn(B, n, H, 64, generator=g).to(dev, torch.bfloat16) for n in (Lq, Lk, Lk))
    d_o = torch.randn(B, Lq, H, 64, generator=g).to(dev, torch.bfloat16)
    return q, k, v, d_o


def _reference(q, k, v, d_o, o, vis, keep, dscale):
    """fp32 O, lse, and dQ, dK, dV as the kernels define the backward (FlashAttention-2, delta = rowsum(dO * O) of the
    given O), one batch entry at a time."""
    outs = {n: [] for n in ("o", "lse", "dq", "dk", "dv")}
    for b in range(q.shape[0]):
        qh, kh, vh, doh, oh = (t[b].float().permute(1, 0, 2) if t is not None else None for t in (q, k, v, d_o, o))
        s = (qh @ kh.transpose(-1, -2)) * SCALE
        if vis is not None:
            s = s.masked_fill(~vis[b], float("-inf"))
        lse = torch.logsumexp(s, -1)
        p = torch.softmax(s, -1)
        kp = keep[b].float() * dscale if keep is not None else 1.0
        outs["o"].append(((p * kp) @ vh).permute(1, 0, 2))
        outs["lse"].append(lse)
        if doh is not None:
            ds = p * ((doh @ vh.transpose(-1, -2)) * kp - (doh * oh).sum(-1, keepdim=True))
            outs["dq"].append(((ds @ kh) * SCALE).permute(1, 0, 2))
            outs["dk"].append(((ds.transpose(-1, -2) @ qh) * SCALE).permute(1, 0, 2))
            outs["dv"].append(((p * kp).transpose(-1, -2) @ doh).permute(1, 0, 2))
    return {n: torch.stack(t) for n, t in outs.items() if t}


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30))


BARS = {"o": 6e-3, "dq": 1e-2, "dk": 1e-2, "dv": 1e-2}


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_wgmma_attention_against_fp32(case, dev, L):
    from dreamvla_b200 import ops
    name, B, H, Lq, Lk, mask, p, backward = case
    g = torch.Generator().manual_seed(B * 7919 + Lq * 31 + Lk)
    vis = _backbone_vis() if mask == "backbone" else _random_vis(Lq, Lk, g) if mask == "random" else None
    am = ops.AttnMask(vis, dev) if vis is not None else None
    bits, flags = (am.bits, am.flags) if am is not None else (None, None)
    if mask == "random" and Lq >= 256 and Lk >= 256:
        assert {0, 1, 2} <= set(flags.flatten().tolist()), "want skipped, partial and full tiles"
    q, k, v, d_o = _inputs(B, H, Lq, Lk, dev, g)

    def run():
        o, lse = L.attn_fwd(q, k, v, SCALE, bits, flags, dropout_p=p, dropout_seed=SEED)
        grads = ()
        if backward:
            dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
            L.attn_bwd(q, k, v, o, d_o, lse, SCALE, dq, dk, dv, bits, flags, dropout_p=p, dropout_seed=SEED)
            grads = (dq, dk, dv)
        return (o, lse) + grads

    first, second = run(), run()
    torch.cuda.synchronize()
    for a, b in zip(first, second):
        assert torch.equal(a, b), f"{name}: two launches differ"
    keep = None
    if p > 0:
        keep = torch.from_numpy(R.keep_attn(SEED, B, H, Lq, Lk, p)).to(dev)
    _, dscale = R.thresh_scale(p) if p > 0 else (0, 1.0)
    visb = vis.to(dev)[None].expand(B, -1, -1)[:, None] if vis is not None else None
    ref = _reference(q, k, v, d_o if backward else None, first[0], visb, keep, dscale)
    got = dict(zip(("o", "lse", "dq", "dk", "dv"), first))
    lse_err = float((got["lse"] - ref["lse"]).abs().max())
    errs = {n: _rel(got[n], ref[n]) for n in BARS if n in ref}
    print(f"[attn-wgmma] {name}: lse {lse_err:.1e} " + " ".join(f"{n} {e:.1e}" for n, e in errs.items()))
    assert lse_err < 1e-3, f"{name}: lse off by {lse_err:.3e}"
    bad = {n: e for n, e in errs.items() if not e < BARS[n]}
    assert not bad, f"{name}: relative L2 error over the bars {BARS}: {bad}"


def test_wgmma_forward_per_sequence_masks(dev, L):
    """A two-mask stack selected per sequence (mask_index) equals each sequence run alone under its own mask, bit for bit,
    and the fp32 reference under that mask."""
    from dreamvla_b200 import ops
    g = torch.Generator().manual_seed(11)
    B, H, Lx = 4, 2, 300
    vis = torch.stack([_random_vis(Lx, Lx, g), _random_vis(Lx, Lx, g)])
    stack = ops.AttnMaskStack(vis, dev)
    index = torch.tensor([1, 0, 0, 1], dtype=torch.int32, device=dev)
    q, k, v, _ = _inputs(B, H, Lx, Lx, dev, g)
    o, lse = L.attn_fwd(q, k, v, SCALE, stack.bits, stack.flags, mask_index=index)
    o2, _ = L.attn_fwd(q, k, v, SCALE, stack.bits, stack.flags, mask_index=index)
    assert torch.equal(o, o2)
    for b in range(B):
        m = ops.AttnMask(vis[int(index[b])], dev)
        ob, lb = L.attn_fwd(q[b:b + 1], k[b:b + 1], v[b:b + 1], SCALE, m.bits, m.flags)
        assert torch.equal(o[b:b + 1], ob) and torch.equal(lse[b:b + 1], lb), f"sequence {b}"
    visb = vis[index.long().cpu()].to(dev)[:, None]
    ref = _reference(q, k, v, None, o, visb, None, 1.0)
    assert _rel(o, ref["o"]) < BARS["o"]
    assert float((lse - ref["lse"]).abs().max()) < 1e-3
