"""Host logic of the GEMM dispatcher, without a GPU: `dvla_gemm_plan` runs the same code as `dvla_gemm` up to the point where
tensor maps would be encoded and the kernel launched, and `dvla_gemm_plan_unit` evaluates the same unit -> (tile, k-range)
map the persistent kernels walk (`map_unit`, shared host/device function in csrc/gemm_sm90.cu).

Checked over the GEMM shapes of the C2 / C3 / C4 workloads, their weight-gradient forms, and a random sweep:
  * every (output tile, k-block) is covered by exactly one work unit -- whole tiles, uniform split-K and the K-split tail;
  * a tail starts on a wave boundary, only exists for GEMMs of at least one full wave (batch-invariance of the sub-wave
    GEMMs of action inference, tests/test_rollout_gpu.py), and its partial tiles fit the workspace;
  * without a workspace there is no tail; pure accumulations (out == residual) may split K, everything else may not;
  * the SM budget (`dvla_set_sm_budget`, lowered while NCCL shares the GPU) resizes grids and moves the wave boundary;
  * every case of the GPU path table (tests/gemm_cases.py) plans the kernel path it declares, at 132 and 114 SMs.
"""
import ctypes as C
import random

import pytest

from dreamvla_b200 import _lib, build
from tests import gemm_cases as GC

FAKE = 0x7F0000000000        # aligned fake device addresses: the planner only tests pointers for NULL / alignment


@pytest.fixture(scope="module")
def lib():
    build.build_library()
    return _lib.load()


def plan(lib, M, N, K, a_mn=False, b_mn=False, accumulate=False, bias=False, act=0, workspace=True, lda=None, ldb=None):
    a = _lib.GemmArgs()
    a.a, a.b, a.out = FAKE, FAKE + (1 << 32), FAKE + (2 << 32)
    a.M, a.N, a.K = M, N, K
    a.lda = lda if lda is not None else (M if a_mn else K)
    a.ldb = ldb if ldb is not None else (N if b_mn else K)
    a.ldo = N
    a.a_mn_major, a.b_mn_major = int(a_mn), int(b_mn)
    a.alpha = 1.0
    a.act = act
    if accumulate:
        a.residual, a.ldr = a.out, N
    if bias:
        a.bias = FAKE + (3 << 32)
    if workspace:
        a.workspace, a.workspace_bytes = FAKE + (4 << 32), int(lib.dvla_gemm_workspace_bytes(None))
    out = _lib.GemmPlanInfo()
    rc = lib.dvla_gemm_plan(C.byref(a), C.byref(out))
    assert rc == 0, lib.dvla_last_error()
    return out


def units(lib, p):
    res = []
    t, k0, k1, slot, split = (C.c_int32() for _ in range(5))
    for u in range(p.units):
        assert lib.dvla_gemm_plan_unit(C.byref(p), u, C.byref(t), C.byref(k0), C.byref(k1), C.byref(slot), C.byref(split)) == 0
        res.append((t.value, k0.value, k1.value, slot.value, split.value))
    return res


def check_cover(lib, p, M, N, K):
    """Every k-block of every tile exactly once; returns the unit list."""
    assert p.kernel == 2
    assert p.m_tiles == -(-M // p.tile_m) and p.n_tiles == -(-N // p.tile_n) and p.k_blocks == -(-K // 64)
    tiles = p.m_tiles * p.n_tiles
    seen = [[0] * p.k_blocks for _ in range(tiles)]
    us = units(lib, p)
    for (t, k0, k1, slot, split) in us:
        assert 0 <= t < tiles and 0 <= k0 < k1 <= p.k_blocks, (t, k0, k1)
        for kb in range(k0, k1):
            seen[t][kb] += 1
    assert all(c == 1 for row in seen for c in row), "a (tile, k-block) is covered zero or several times"
    return us


def check_tail(lib, p, us, slots_per_wave):
    tiles = p.m_tiles * p.n_tiles
    if p.tail_splits <= 1:
        assert all(slot < 0 for (_, _, _, slot, _) in us)
        return
    assert p.k_splits == 1 and not p.atomic_out
    assert p.tail_first >= slots_per_wave and p.tail_first % slots_per_wave == 0, "the tail must start on a wave boundary, after >= 1 full wave"
    n_tail = tiles - p.tail_first
    assert 0 < n_tail < slots_per_wave and n_tail * p.tail_splits <= slots_per_wave, "the split tail must fit one wave"
    for u, (t, k0, k1, slot, split) in enumerate(us):
        if u < p.tail_first:
            assert (t, k0, k1, slot) == (u, 0, p.k_blocks, -1)
        else:
            assert slot == t - p.tail_first and 0 <= split < p.tail_splits and k0 == split * p.tail_kbps
    # workspace: 64 KB of counters (8 per CTA slot) + one fp32 slice of 128 x tile_n per CTA slot and split
    need = 65536 + n_tail * p.tail_splits * 128 * p.tile_n * 4
    assert need <= int(lib.dvla_gemm_workspace_bytes(None)) and n_tail * 8 * 4 <= 65536


WORKLOAD = [  # (M, N, K, b_mn)  forward / dgrad GEMMs of C2 at B=8 and B=2, C3 at B=16, C4 (action inference)
    (10320, 1024, 4096, True), (10320, 4096, 1024, True), (10320, 3072, 1024, True), (10320, 1024, 1024, True),
    (10320, 1024, 4096, False), (10320, 1024, 3072, False), (32800, 4096, 1024, False), (32800, 1024, 4096, False),
    (42400, 4096, 1024, False), (42400, 1024, 4096, False), (31520, 3072, 768, False), (31520, 768, 3072, False),
    (31520, 2304, 768, False), (2580, 1024, 4096, True), (2580, 4096, 1024, True), (2580, 3072, 1024, True),
    (4368, 1024, 4096, True), (930, 1024, 4096, True), (930, 4096, 1024, True), (129, 1024, 4096, True), (21, 768, 3072, False),
    (12, 3072, 768, False), (394, 768, 3072, False), (3940, 3072, 768, False),
]


@pytest.mark.parametrize("sms", [132, 116])
def test_workload_gemms_are_covered_exactly_once(lib, sms):
    lib.dvla_set_sm_budget(sms)
    try:
        for (M, N, K, b_mn) in WORKLOAD:
            p = plan(lib, M, N, K, b_mn=b_mn, bias=True)
            us = check_cover(lib, p, M, N, K)
            check_tail(lib, p, us, sms)
            assert p.grid_ctas <= sms and p.k_splits == 1 and not p.atomic_out, "a GEMM with an epilogue never splits K uniformly"
            tiles = p.m_tiles * p.n_tiles
            if tiles < sms:
                assert p.tail_splits <= 1, "sub-wave GEMMs keep one K order whatever the batch (batch invariance)"
    finally:
        lib.dvla_set_sm_budget(0)


def test_known_decisions(lib):
    lib.dvla_set_sm_budget(0)
    p = plan(lib, 2580, 1024, 4096, b_mn=True, bias=True)           # 21 x 8 = 168 tiles on 132 SMs: 1 wave + 36
    assert (p.kernel, p.tile_m, p.tile_n, p.tail_first, p.tail_splits, p.tail_kbps) == (2, 128, 128, 132, 3, 22)
    assert p.units == 132 + 36 * 3 and p.grid_ctas == 132
    p = plan(lib, 2580, 1024, 1024, b_mn=True, bias=True)           # 16 k-blocks: the fix-up would cost more than the wave
    assert p.tail_splits <= 1
    p = plan(lib, 2580, 1024, 4096, b_mn=True, bias=True, workspace=False)
    assert p.tail_splits <= 1 and p.units == 168
    p = plan(lib, 21, 7, 768, bias=True, ldb=768)                   # N = 7: TMA-addressable operands but a 7-wide output
    assert p.kernel in (0, 1, 2)
    p = plan(lib, 21, 768, 6, lda=6, ldb=6)                         # K = 6: rows are not 16-byte multiples -> SIMT kernel
    assert p.kernel in (0, 1)


def test_weight_gradient_split_k(lib):
    """G[M,N] += A^T B with K = B*S*tokens: few output tiles, a very long contraction -> uniform split-K with bf16 atomics,
    never the K-split tail."""
    lib.dvla_set_sm_budget(0)
    for (M, N, K) in [(1024, 1024, 10320), (4096, 1024, 10320), (1024, 3072, 10320), (768, 3072, 31520), (1024, 4096, 42400),
                      (520, 264, 4104), (128, 136, 2056)]:
        p = plan(lib, M, N, K, a_mn=True, b_mn=True, accumulate=True)
        check_cover(lib, p, M, N, K)
        assert p.tail_splits <= 1
        if p.k_splits > 1:
            assert p.atomic_out == 1 and p.kb_per_split * p.k_splits >= p.k_blocks > p.kb_per_split * (p.k_splits - 1)
        tiles = p.m_tiles * p.n_tiles
        slots = 132
        if K >= 10320 and tiles * 2 <= slots:
            assert max(p.k_splits, p.tail_splits) > 1, "a long contraction over a few tiles must be split"


def test_random_shapes(lib):
    rng = random.Random(7)
    lib.dvla_set_sm_budget(0)
    for _ in range(300):
        M = rng.choice([rng.randrange(1, 300), rng.randrange(300, 5000), rng.randrange(5000, 45000)])
        N = 8 * rng.randrange(1, 520)
        K = 8 * rng.randrange(1, 700)
        b_mn = rng.random() < 0.5
        accumulate = rng.random() < 0.2
        p = plan(lib, M, N, K, b_mn=b_mn, accumulate=accumulate, bias=not accumulate, ldb=(N if b_mn else K))
        if p.kernel < 2:
            continue
        us = check_cover(lib, p, M, N, K)
        if not accumulate:
            check_tail(lib, p, us, 132)
            assert p.k_splits == 1


def plan_case(lib, c):
    """dvla_gemm_plan of a tests/gemm_cases.py case, with fake pointers offset like the case's matrices."""
    esz = 4 if c.out_fp32 else 2
    a = _lib.GemmArgs()
    a.a, a.b = FAKE + 2 * c.a_off, FAKE + (1 << 32) + 2 * c.b_off
    a.out = FAKE + (2 << 32) + esz * c.out_off
    a.M, a.N, a.K = c.M, c.N, c.K
    a.lda, a.ldb, a.ldo = c.lda, c.ldb, c.ldo
    a.a_mn_major, a.b_mn_major = int(c.a_mn), int(c.b_mn)
    a.act, a.out_fp32, a.alpha = c.act, int(c.out_fp32), c.alpha
    if c.has_bias:
        a.bias = FAKE + (3 << 32)
    if c.residual_is_out:
        a.residual, a.ldr = a.out, c.ldo
    elif c.has_residual:
        a.residual, a.ldr = FAKE + (5 << 32) + esz * c.res_off, c.ldr
    if c.recipe == "full":
        a.aux_out, a.ld_aux = FAKE + (6 << 32) + 2 * c.aux_off, c.ld_aux
    elif c.recipe == "dgrad":
        a.aux_in, a.ld_aux = FAKE + (6 << 32) + 2 * c.aux_off, c.ld_aux
    if c.recipe == "dropout":
        a.dropout_p, a.dropout_seed_ptr = GC.DROPOUT_P, FAKE + (7 << 32)
    a.workspace, a.workspace_bytes = FAKE + (4 << 32), int(lib.dvla_gemm_workspace_bytes(None))
    out = _lib.GemmPlanInfo()
    assert lib.dvla_gemm_plan(C.byref(a), C.byref(out)) == 0, lib.dvla_last_error()
    return out


@pytest.mark.parametrize("sms", GC.SM_BUDGETS)
def test_case_table_paths(lib, sms):
    """Every case of tests/gemm_cases.py reaches the path it declares, at the SM counts of the H100 SXM and PCIe; and the
    table covers every path with every reachable majorness x recipe, and every activation on a staged and a direct path."""
    lib.dvla_set_sm_budget(sms)
    try:
        wrong = []
        for c in GC.CASES:
            got = GC.path_of(plan_case(lib, c), c)
            if got != c.path_at(sms):
                wrong.append(f"{c.id}: plans {got}")
        assert not wrong, f"{len(wrong)} cases leave their declared path at {sms} SMs:\n" + "\n".join(wrong[:20])
    finally:
        lib.dvla_set_sm_budget(0)
    have = {(c.path, c.a_mn, c.b_mn, c.recipe) for c in GC.CASES}
    for path in GC.PATHS:
        recipes = {"wgmma_splitk": ("accum",), "wgmma_tail": ("plain", "full", "dgrad", "dropout")}.get(path, GC.RECIPES)
        missing = [(path, a, b, r) for (a, b) in GC.MAJORS for r in recipes if (path, a, b, r) not in have]
        assert not missing, missing
    acts = {(c.path in GC.STAGED_PATHS, c.act) for c in GC.CASES if c.recipe in ("full", "dgrad", "dropout")}
    assert all((staged, act) in acts for staged in (True, False) for act in range(6)), sorted(acts)
