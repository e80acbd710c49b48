"""The persistent schedule of the wgmma attention backward (attn_bwd_wgmma_kernel): each CTA walks work units (b, h, pair of
fixed tiles) with a stride of the grid, and the producer loads the next unit's tiles while the consumers finish the
current one.  These cases reach what the shapes of test_attn_wgmma_gpu.py do not: more units than CTAs at an odd tile
count (a lone last tile in every (b, h)), fewer units than SMs with a single (b, h), and a grid cut down by the SM budget
(dvla_set_sm_budget, lowered while a collective shares the GPU).  Each is checked against fp32 torch, for the same bits
across two launches, and (budget) for the same bits as the full-width grid."""
import pytest
import torch

from tests import philox_ref as R
from tests.test_attn_wgmma_gpu import BARS, SCALE, SEED, _backbone_vis, _inputs, _random_vis, _reference, _rel

pytestmark = pytest.mark.gpu


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


# (id, B, H, L, mask, p, SM budget or 0)
CASES = [
    ("odd_tiles_40x8x300_random_p0.1", 40, 8, 300, "random", 0.1, 0),     # 5 tiles: 3 units per (b, h), 960 units
    ("single_bh_1x1x1290_backbone_p0.1", 1, 1, 1290, "backbone", 0.1, 0),  # 11 units, far fewer than SMs
    ("budget40_24x16x265_p0.1", 24, 16, 265, None, 0.1, 40),               # 1152 units on 40 CTAs
    ("budget10_odd_3x5x330_random_p0", 3, 5, 330, "random", 0.0, 10),
]


def _run(L, q, k, v, d_o, bits, flags, p):
    o, lse = L.attn_fwd(q, k, v, SCALE, bits, flags, dropout_p=p, dropout_seed=SEED)
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    L.attn_bwd(q, k, v, o, d_o, lse, SCALE, dq, dk, dv, bits, flags, dropout_p=p, dropout_seed=SEED)
    torch.cuda.synchronize()
    return o, dq, dk, dv


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_attn_bwd_schedule(case, dev, L):
    from dreamvla_b200 import ops
    name, B, H, Lx, mask, p, budget = case
    g = torch.Generator().manual_seed(B * 7919 + Lx * 31 + H)
    vis = _backbone_vis() if mask == "backbone" else _random_vis(Lx, Lx, g) if mask == "random" else None
    am = ops.AttnMask(vis, dev) if vis is not None else None
    bits, flags = (am.bits, am.flags) if am is not None else (None, None)
    q, k, v, d_o = _inputs(B, H, Lx, Lx, dev, g)

    full = _run(L, q, k, v, d_o, bits, flags, p) if budget else None
    prev = L.set_sm_budget(budget) if budget else None
    try:
        first = _run(L, q, k, v, d_o, bits, flags, p)
        second = _run(L, q, k, v, d_o, bits, flags, p)
    finally:
        if budget:
            L.set_sm_budget(prev)
    for n, a, b in zip(("o", "dq", "dk", "dv"), first, second):
        assert torch.equal(a, b), f"{name}: two launches differ in {n}"
        if full is not None:
            assert torch.equal(a, full[("o", "dq", "dk", "dv").index(n)]), f"{name}: {n} differs from the full-width grid"

    keep = torch.from_numpy(R.keep_attn(SEED, B, H, Lx, Lx, p)).to(dev) if p > 0 else None
    _, dscale = R.thresh_scale(p) if p > 0 else (0, 1.0)
    visb = vis.to(dev)[None].expand(B, -1, -1)[:, None] if vis is not None else None
    ref = _reference(q, k, v, d_o, first[0], visb, keep, dscale)
    errs = {n: _rel(t, ref[n]) for n, t in zip(("dq", "dk", "dv"), first[1:])}
    print(f"[attn-bwd-schedule] {name}: " + " ".join(f"{n} {e:.1e}" for n, e in errs.items()))
    bad = {n: e for n, e in errs.items() if not e < BARS[n]}
    assert not bad, f"{name}: relative L2 error over the bars {BARS}: {bad}"
