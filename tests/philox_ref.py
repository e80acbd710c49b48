"""Host restatement (numpy) of the library's dropout RNG, so that every dropout mask the kernels draw can be recomputed bit
for bit and the dropout kernels tested against plain references evaluated under the same mask.

What it restates (csrc/common.cuh `philox4x32` / `dropout_keep8`, include/dvla.h):
  * Philox-4x32 (Salmon et al., SC'11) with counter (offset_lo, offset_hi, 0x243F6A88, 0x85A308D3) and key (seed_lo,
    seed_hi); the kernels run 7 rounds.  All arithmetic is mod 2^32 per word.
  * one Philox call = one RNG block of 8 elements; element j of the block draws the low (j even) or high (j odd) 16 bits of
    word j // 2 and is kept iff that draw >= thresh.
  * GEMM epilogue / dvla_dropout: block = m * ceil(N / 8) + n / 8, bit n % 8.
    Attention probabilities:       block = ((b * H + h) * Lq + i) * ceil(Lk / 8) + j / 8, bit j % 8.
  * thresh = (uint32)(p * 65536.0f + 0.5f), scale = 1 / (1 - thresh / 65536.0f), both in fp32 on the host.
  * effective seed = seed + *seed_ptr (the device counter), mod 2^64.
"""
from __future__ import annotations

import numpy as np

ROUNDS = 7
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
_C2, _C3 = 0x243F6A88, 0x85A308D3
_LO = np.uint64(0xFFFFFFFF)
_U64 = (1 << 64) - 1


def philox4x32(ctr, key, rounds=ROUNDS):
    """Philox-4x32-`rounds` of counter words ctr[0..3] under key words key[0..1] (ints or uint64 arrays of 32-bit values,
    broadcast together) -> four uint64 arrays of 32-bit output words."""
    c0, c1, c2, c3 = (np.asarray(x, dtype=np.uint64) & _LO for x in ctr)
    k0, k1 = (np.asarray(x, dtype=np.uint64) & _LO for x in key)
    for _ in range(rounds):
        p0 = _M0 * c0                     # 32 x 32 -> 64-bit product: hi word = __umulhi, lo word = the 32-bit product
        p1 = _M1 * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _LO, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _LO
        k0 = (k0 + _W0) & _LO
        k1 = (k1 + _W1) & _LO
    return c0, c1, c2, c3


def thresh_scale(p):
    """(thresh, scale) exactly as the library rounds them from a float32 `p` (dropout_thresh_scale, csrc/host.cuh)."""
    pf = np.float32(p)
    thresh = int(np.uint32(pf * np.float32(65536.0) + np.float32(0.5)))
    scale = np.float32(1.0) / (np.float32(1.0) - np.float32(thresh) / np.float32(65536.0))
    return thresh, float(scale)


def keep_blocks(seed, blocks, p):
    """Keep bits of RNG blocks `blocks` (uint64 array) under effective seed `seed`: bool [*blocks.shape, 8]."""
    seed = int(seed) & _U64
    thresh, _ = thresh_scale(p)
    blocks = np.asarray(blocks, dtype=np.uint64)
    w = philox4x32((blocks & _LO, blocks >> np.uint64(32), _C2, _C3), (seed & 0xFFFFFFFF, seed >> 32))
    halves = np.stack([h for x in w for h in (x & np.uint64(0xFFFF), x >> np.uint64(16))], axis=-1)
    return halves >= np.uint64(thresh)


def keep_rows(seed, rows, N, p, counter=0):
    """GEMM-epilogue / dvla_dropout mask of a [rows, N] output: bool [rows, N] (True = kept)."""
    nblk = (N + 7) // 8
    blocks = np.arange(rows * nblk, dtype=np.uint64).reshape(rows, nblk)
    return keep_blocks(int(seed) + int(counter), blocks, p).reshape(rows, nblk * 8)[:, :N]


def keep_attn(seed, B, H, Lq, Lk, p, counter=0):
    """Attention-probability mask of a [B, H, Lq, Lk] score tensor: bool [B, H, Lq, Lk] (True = kept)."""
    return keep_rows(seed, B * H * Lq, Lk, p, counter).reshape(B, H, Lq, Lk)
