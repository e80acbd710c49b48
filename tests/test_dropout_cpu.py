"""The host restatement of the dropout RNG (tests/philox_ref.py), without a GPU: Philox-4x32 against Random123's published
known-answer vectors, the fp32 rounding of (thresh, scale), and the statistics of the 7-round masks the kernels draw."""
import numpy as np
import pytest
import torch

from tests import philox_ref as R

# Random123 kat_vectors, philox4x32-10: (counter, key, expected output)
KAT = [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(w) for w in R.philox4x32(ctr, key, rounds=10)) == want


def test_philox_vectorised_equals_scalar():
    rng = np.random.default_rng(0)
    ctr = [rng.integers(0, 2 ** 32, 64, dtype=np.uint64) for _ in range(4)]
    key = [rng.integers(0, 2 ** 32, 64, dtype=np.uint64) for _ in range(2)]
    vec = R.philox4x32(ctr, key)
    for i in range(64):
        one = R.philox4x32([c[i] for c in ctr], [k[i] for k in key])
        assert tuple(int(w) for w in one) == tuple(int(v[i]) for v in vec)


def _fp32(x):
    return torch.tensor(x, dtype=torch.float32)


@pytest.mark.parametrize("p,thresh", [(1e-6, 0), (0.1, 6554), (0.5, 32768), (0.9, 58982), (0.99999, 65535)])
def test_thresh_scale_rounding(p, thresh):
    t, s = R.thresh_scale(p)
    assert t == thresh
    # the dispatchers' arithmetic, restated with torch fp32 tensors: thresh = (uint32)(p * 65536.0f + 0.5f), scale = 1 / (1 - t / 65536.0f)
    assert int(_fp32(p) * 65536.0 + 0.5) == thresh
    want = (_fp32(1.0) / (_fp32(1.0) - _fp32(float(thresh)) / _fp32(65536.0))).item()
    assert s == want
    if thresh == 0:
        assert s == 1.0


def test_keep_rows_layout():
    """Row r of a [rows, N] mask is blocks r*ceil(N/8) .. ; bit n%8 of block n/8; the padding bits past N are dropped."""
    seed, p, N = 0x0123456789ABCDEF, 0.3, 13
    m = R.keep_rows(seed, 5, N, p)
    assert m.shape == (5, N)
    blocks = R.keep_blocks(seed, np.arange(10, dtype=np.uint64), p)
    for r in range(5):
        assert np.array_equal(m[r], np.concatenate([blocks[2 * r], blocks[2 * r + 1]])[:N])
    # the counter adds to the seed mod 2^64
    assert np.array_equal(R.keep_rows(2 ** 64 - 3, 5, N, p, counter=5), R.keep_rows(2, 5, N, p))
    a = R.keep_attn(seed, 2, 3, 4, N, p)
    assert np.array_equal(a.reshape(24, N), R.keep_rows(seed, 24, N, p))


def test_keep_rate_per_bit_position():
    n = 1 << 20
    for p in (0.1, 0.5):
        thresh, _ = R.thresh_scale(p)
        q = 1.0 - thresh / 65536.0
        bits = R.keep_blocks(0x9E3779B97F4A7C15, np.arange(n, dtype=np.uint64) + np.uint64(3 << 40), p)
        sigma = np.sqrt(q * (1 - q) / n)
        rate = bits.mean(axis=0)
        assert np.all(np.abs(rate - q) < 5 * sigma), (p, rate, q)


def _corr(a, b):
    a, b = a.astype(np.float64).ravel(), b.astype(np.float64).ravel()
    return float(np.corrcoef(a, b)[0, 1]), 1.0 / np.sqrt(a.size)


def test_adjacent_seeds_uncorrelated():
    """The train step advances the device seed counter by exactly 1 per micro-step, so the masks of seeds s and s+1 must be
    independent (a weak key schedule would correlate them)."""
    for s in (0, 0x243F6A8885A308D3, 2 ** 64 - 1):
        m0 = R.keep_rows(s, 1024, 1024, 0.1)
        m1 = R.keep_rows(s, 1024, 1024, 0.1, counter=1)
        c, sigma = _corr(m0, m1)
        assert abs(c) < 5 * sigma, (s, c, sigma)


def test_adjacent_heads_uncorrelated():
    """Adjacent (b, h) rows of one attention call use consecutive block ranges of one seed."""
    m = R.keep_attn(0x5851F42D4C957F2D, 2, 2, 512, 512, 0.1)
    for (b0, h0), (b1, h1) in (((0, 0), (0, 1)), ((0, 1), (1, 0)), ((1, 0), (1, 1))):
        c, sigma = _corr(m[b0, h0], m[b1, h1])
        assert abs(c) < 5 * sigma, ((b0, h0), (b1, h1), c, sigma)
    # and neighbouring query rows of one head
    c, sigma = _corr(m[0, 0, :-1], m[0, 0, 1:])
    assert abs(c) < 5 * sigma


@pytest.mark.parametrize("p", [float("nan"), 1.0, 1.5, -0.25])
def test_gemm_rejects_out_of_range_dropout_p(p):
    """dvla_gemm_plan runs dvla_gemm's argument checks without a GPU: a NaN or out-of-range rate is an error, not a
    silently disabled (NaN > 0 is false) or infinite-scale dropout."""
    import ctypes as C
    from dreamvla_b200 import _lib, build
    build.build_library()
    lib = _lib.load()
    fake = 0x7F0000000000
    a = _lib.GemmArgs()
    a.a, a.b, a.out = fake, fake + (1 << 32), fake + (2 << 32)
    a.M, a.N, a.K, a.lda, a.ldb, a.ldo = 256, 256, 256, 256, 256, 256
    a.alpha, a.dropout_p = 1.0, p
    info = _lib.GemmPlanInfo()
    assert lib.dvla_gemm_plan(C.byref(a), C.byref(info)) == -1
    assert b"dropout_p" in lib.dvla_last_error()
    a.dropout_p = 0.1
    assert lib.dvla_gemm_plan(C.byref(a), C.byref(info)) == 0
