// Flash-style multi-head attention for head_dim = 64 with a bit-matrix visibility mask and tile skipping.  The entry points
// also route the short-sequence case (head_dim 64 or 96) to attention_small.cu.
//
// Data path of the mma.sync kernels: cp.async -> XOR-swizzled smem tiles -> ldmatrix -> mma.sync.m16n8k16 (bf16, fp32 accumulate),
// online softmax in registers, no [Lq,Lk] tensor in HBM.  These serve short query blocks and strides a tensor map cannot
// express; long sequences (>= 96) run on the TMA + wgmma warp-specialised kernels further down (attn_fwd_wgmma_kernel,
// attn_bwd_wgmma_kernel), the short unmasked ones of the DiT on attention_small.cu.
//
// Kernels:
//   attn_fwd_kernel     grid (ceil(Lq/64), H, B), 4 warps x 16 query rows, K/V tiles of 64 keys double-buffered
//   attn_delta_kernel   delta[b,h,i] = sum_d dO*O
//   attn_bwd_dkv_kernel grid (ceil(Lk/64), H, B): per key tile, loops over query tiles, S^T/dP^T formulation
//   attn_bwd_dq_kernel  grid (ceil(Lq/64), H, B): per query tile, loops over key tiles
// Masking: tile_flags[qt, kt] in {0 skip, 1 partial, 2 full}; partial tiles test bits of mask[i, j/32].
// Both kernel families share the per-fragment helpers below dropout_bits: mask words, the forward tile step, the dQ-form dS
// and the scaled bf16 store.  The forward finish and the dK/dV-form P / dS^T stay written out per kernel (see there).
#include <limits.h>
#include <string.h>

#include <mutex>

#include "common.cuh"
#include "host.cuh"
#include "../../include/dvla.h"

namespace dvla {

constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

struct AttnParams {
  const bf16 *q, *k, *v, *o, *d_o;
  bf16 *out, *dq, *dk, *dv;
  float* lse;
  float* delta;
  const uint32_t* mask;
  const uint8_t* tile_flags;
  int B, H, Lq, Lk, nqt, nkt, mask_words;
  long long q_sb, q_ss, q_sh, k_sb, k_ss, k_sh, v_sb, v_ss, v_sh, o_sb, o_ss, o_sh;
  long long do_sb, do_ss, do_sh, dq_sb, dq_ss, dq_sh, dk_sb, dk_ss, dk_sh, dv_sb, dv_ss, dv_sh;
  float scale;
  float drop_scale; uint32_t drop_thresh; uint64_t drop_seed; const uint64_t* drop_seed_ptr;
  // forward with per-sequence masks (PER_SEQ kernels): batch b reads mask / tile_flags advanced by mask_index[b] strides
  const int32_t* mask_index; long long mask_stride, flags_stride;
};

// ---- smem tile helpers: 64 rows x 64 bf16 (128 B per row), 16-byte chunk c of row r stored at chunk c ^ (r & 7) --------
__device__ __forceinline__ uint32_t tile_addr(uint32_t base, int row, int chunk) {
  return base + row * 128 + ((chunk ^ (row & 7)) << 4);
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// rows [r0, r0+64) of a strided [L, 64] matrix -> swizzled tile; rows >= L are zero-filled.  128 threads.
__device__ __forceinline__ void load_tile_async(uint32_t sbase, const bf16* g, long long row_stride, int r0, int L) {
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int i = threadIdx.x + it * 128;
    const int row = i >> 3, ch = i & 7;
    const int gr = r0 + row;
    const bf16* src = g + static_cast<long long>(gr < L ? gr : (L - 1)) * row_stride + ch * 8;
    cp_async16(tile_addr(sbase, row, ch), src, gr < L ? 16 : 0);
  }
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// A fragments (16 rows x 64 cols) of a tile for this warp's 16 rows starting at row r0: frag[kk][0..3]
__device__ __forceinline__ void load_a_frags(uint32_t tile, int r0, uint32_t (&f)[4][4]) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) ldsm_x4(tile_addr(tile, r0 + (lane & 15), kk * 2 + (lane >> 4)), f[kk]);
}
// C[16 x 64] (+)= A[16 x 64(k)] * T^T where T is a [64(n) x 64(k)] row-major tile (B fragment = plain ldmatrix)
__device__ __forceinline__ void mma_a_tT(float (&c)[8][4], const uint32_t (&a)[4][4], uint32_t tile) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      uint32_t b[4];
      ldsm_x4(tile_addr(tile, np * 16 + (lane & 7) + ((lane >> 4) << 3), kk * 2 + ((lane >> 3) & 1)), b);
      mma16816(c[2 * np], a[kk], b[0], b[1]);
      mma16816(c[2 * np + 1], a[kk], b[2], b[3]);
    }
  }
}
// C[16 x 64(n)] += P[16 x 64(k)] * T where T is a [64(k) x 64(n)] row-major tile (B fragment = ldmatrix.trans);
// P given as packed bf16 A fragments pa[kk][0..3].
__device__ __forceinline__ void mma_p_t(float (&c)[8][4], const uint32_t (&pa)[4][4], uint32_t tile) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      uint32_t b[4];
      ldsm_x4_t(tile_addr(tile, kk * 16 + (lane & 7) + (((lane >> 3) & 1) << 3), np * 2 + (lane >> 4)), b);
      mma16816(c[2 * np], pa[kk], b[0], b[1]);
      mma16816(c[2 * np + 1], pa[kk], b[2], b[3]);
    }
  }
}
// C-fragment layout (16 x 64 fp32) -> A-fragment layout (bf16) for the next MMA
__device__ __forceinline__ void c_to_a(const float (&c)[8][4], uint32_t (&a)[4][4]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    a[kk][0] = pack_bf16x2(c[2 * kk][0], c[2 * kk][1]);
    a[kk][1] = pack_bf16x2(c[2 * kk][2], c[2 * kk][3]);
    a[kk][2] = pack_bf16x2(c[2 * kk + 1][0], c[2 * kk + 1][1]);
    a[kk][3] = pack_bf16x2(c[2 * kk + 1][2], c[2 * kk + 1][3]);
  }
}
__device__ __forceinline__ void zero_c(float (&c)[8][4]) {
#pragma unroll
  for (int t = 0; t < 8; ++t)
#pragma unroll
    for (int e = 0; e < 4; ++e) c[t][e] = 0.f;
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// Dropout keep bits for this thread's elements of a 16x64 C fragment whose rows are `grow0 + {g, g+8}` and whose
// columns are `gcol0 + t*8 + 2c + {0,1}`; RNG block = (bh*Lrow + grow) * ceil(Lcol/8) + gcol/8 (8 consecutive columns).
// The 4 lanes of a quad split the 16 (row, n-tile) Philox calls and exchange 8-bit masks by shuffle.
// `transposed`: fragment holds S^T (rows are keys, cols are queries) -> (row,col) swap for the index.
__device__ __forceinline__ void dropout_bits(const AttnParams& p, long long bh, int frag_row0, int frag_col0,
                                             bool transposed, uint32_t (&keep)[8] /* per n-tile: 4 bits e0..e3 */) {
  const int lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
  const int nblk = (p.Lk + 7) >> 3;
  const uint64_t seed = p.drop_seed + (p.drop_seed_ptr ? __ldg(p.drop_seed_ptr) : 0ull);
  if (!transposed) {
    // rows = queries, cols = keys: one RNG block == one n-tile of one row.
    uint32_t m[2][2];
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int t = c + half * 4;
        const long long row = frag_row0 + g + r * 8;
        m[r][half] = dropout_keep8(seed, (bh * p.Lq + row) * nblk + ((frag_col0 >> 3) + t), p.drop_thresh);
      }
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int src = (lane & ~3) | (t & 3);
      const uint32_t m0 = __shfl_sync(0xffffffffu, m[0][t >> 2], src);
      const uint32_t m1 = __shfl_sync(0xffffffffu, m[1][t >> 2], src);
      keep[t] = ((m0 >> (2 * c)) & 3u) | (((m1 >> (2 * c)) & 3u) << 2);
    }
  } else {
    // rows = keys, cols = queries: a block holds 8 keys of one query, and keys g and g+8 lie in different blocks, so each
    // of a thread's 32 elements draws its own block.  Element (key kr, query qc): block (bh*Lq + qc) * nblk + kr/8, bit kr%8.
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      uint32_t bits = 0;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int kr = frag_row0 + g + (e >> 1) * 8;
        const long long qc = frag_col0 + t * 8 + 2 * c + (e & 1);
        const uint32_t mk = dropout_keep8(seed, (bh * p.Lq + qc) * nblk + (kr >> 3), p.drop_thresh);
        bits |= ((mk >> (kr & 7)) & 1u) << e;
      }
      keep[t] = bits;
    }
  }
}

// ---- per-fragment attention math, shared by the mma.sync and the wgmma kernels -----------------------------------------
// A warp's 16 x 64 fp32 fragment f[t][e] -- an mma.sync C fragment, or the warp's part of a wgmma m64n64 accumulator, which
// has the same layout (common.cuh) -- holds row row0 + lane/4 + 8*(e/2), column col0 + 8t + 2*(lane%4) + e%2.
// sc = scale * log2(e) is passed in: the callers compute it once before their tile loop (computed per tile inside
// fwd_tile_step, it made the wgmma forward ~1.5% slower at the ViT shape on an H100).

// Mask words of the query rows row0 + lane/4 + {0, 8} over keys [k0, k0 + 64): all ones unless the tile is partial (flag 1).
// `mask` is p.mask, or the batch's matrix of a per-sequence stack.
__device__ __forceinline__ void row_mask_words(const AttnParams& p, const uint32_t* mask, int row0, int k0, int flag,
                                               uint32_t (&w)[2][2]) {
  const int g = (threadIdx.x & 31) >> 2;
  w[0][0] = w[0][1] = w[1][0] = w[1][1] = 0xffffffffu;
  if (flag != 1) return;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row0 + g + r * 8;
#pragma unroll
    for (int ww = 0; ww < 2; ++ww) {
      const int wi = (k0 >> 5) + ww;
      w[r][ww] = (row < p.Lq && wi < p.mask_words) ? mask[static_cast<long long>(row) * p.mask_words + wi] : 0u;
    }
  }
}

// Forward step over the key tile [k0, k0 + 64) on S = Q K^T (rows = queries from row0): hide the keys the mask (flag 1) or
// the sequence end hides, scale by sc into the log2 domain, fold the tile into the online softmax (m_run, l_run, o
// rescaled) and drop elements of P.  Leaves P in s.
__device__ __forceinline__ void fwd_tile_step(const AttnParams& p, const uint32_t* mask, float sc, long long bh, int row0,
                                              int k0, int flag, float (&s)[8][4], float (&o)[8][4], float (&m_run)[2],
                                              float (&l_run)[2]) {
  const int c = threadIdx.x & 3;
  const bool tail = (k0 + 64 > p.Lk);
  uint32_t w[2][2];
  row_mask_words(p, mask, row0, k0, flag, w);
  float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int t = 0; t < 8; ++t) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int r = e >> 1;
      const int kk = t * 8 + 2 * c + (e & 1);
      bool vis = true;
      if (flag == 1) vis = (w[r][kk >> 5] >> (kk & 31)) & 1u;
      if (tail) vis = vis && (k0 + kk < p.Lk);
      const float v = vis ? s[t][e] * sc : -INFINITY;
      s[t][e] = v;
      tmax[r] = fmaxf(tmax[r], v);
    }
  }
  float alpha[2], muse[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const float mn = fmaxf(m_run[r], quad_max(tmax[r]));
    muse[r] = (mn == -INFINITY) ? 0.f : mn;
    alpha[r] = exp2f(m_run[r] - muse[r]);
    m_run[r] = mn;
    l_run[r] *= alpha[r];
  }
#pragma unroll
  for (int t = 0; t < 8; ++t) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int r = e >> 1;
      const float pv = exp2f(s[t][e] - muse[r]);
      s[t][e] = pv;
      l_run[r] += pv;
      o[t][e] *= alpha[r];
    }
  }
  if (p.drop_scale != 0.f) {
    uint32_t keep[8];
    dropout_bits(p, bh, row0, k0, false, keep);
#pragma unroll
    for (int t = 0; t < 8; ++t)
#pragma unroll
      for (int e = 0; e < 4; ++e) s[t][e] = ((keep[t] >> e) & 1u) ? s[t][e] * p.drop_scale : 0.f;
  }
}

// lse * log2(e) and delta of the query rows row0 + lane/4 + {0, 8}; +inf and 0 past Lq, so that those rows get P = 0.
__device__ __forceinline__ void row_lse_delta(const AttnParams& p, long long bh, int row0, float (&lse2)[2], float (&dlt)[2]) {
  const int g = (threadIdx.x & 31) >> 2;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row0 + g + r * 8;
    lse2[r] = (row < p.Lq) ? p.lse[bh * p.Lq + row] * LOG2E : INFINITY;
    dlt[r] = (row < p.Lq) ? p.delta[bh * p.Lq + row] : 0.f;
  }
}

// The mask words and dropout keep bits of this thread's query rows over the key tile [k0, k0 + 64), as dq_ds_cols reads them.
struct DqTileBits { uint32_t w[2][2], keep[8]; };
__device__ __forceinline__ void dq_tile_bits(const AttnParams& p, long long bh, int row0, int k0, int flag, DqTileBits& tb) {
  row_mask_words(p, p.mask, row0, k0, flag, tb.w);
  if (p.drop_scale != 0.f) dropout_bits(p, bh, row0, k0, false, tb.keep);
}
// dS = P o (dP - delta) in fragment columns [t0, t1) of the key tile [k0, k0 + 64), rows = queries with their
// row_lse_delta: P recomputed from the LSE and sc, dP dropped with the forward's mask.  Leaves dS in s.
__device__ __forceinline__ void dq_ds_cols(const AttnParams& p, float sc, int k0, const float (&lse2)[2],
                                           const float (&dlt)[2], const DqTileBits& tb, float (&s)[8][4],
                                           const float (&dp)[8][4], int t0, int t1) {
  const int c = threadIdx.x & 3;
#pragma unroll
  for (int t = t0; t < t1; ++t) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int r = e >> 1;
      const int kk = t * 8 + 2 * c + (e & 1);
      // tb.w is all ones outside partial tiles; a hidden key's exponent is -inf, so P is +0 without a branch
      const bool vis = (k0 + kk < p.Lk) && ((tb.w[r][kk >> 5] >> (kk & 31)) & 1u);
      const float pv = exp2f(vis ? s[t][e] * sc - lse2[r] : -INFINITY);
      float dpv = dp[t][e];
      if (p.drop_scale != 0.f) dpv = ((tb.keep[t] >> e) & 1u) ? dpv * p.drop_scale : 0.f;
      s[t][e] = pv * (dpv - dlt[r]);
    }
  }
}
// dq_ds_cols over the whole key tile.
__device__ __forceinline__ void dq_form_ds(const AttnParams& p, float sc, long long bh, int row0, int k0, int flag,
                                           const float (&lse2)[2], const float (&dlt)[2], float (&s)[8][4],
                                           const float (&dp)[8][4]) {
  DqTileBits tb;
  dq_tile_bits(p, bh, row0, k0, flag, tb);
  dq_ds_cols(p, sc, k0, lse2, dlt, tb, s, dp, 0, 8);
}

// Rows row0 + lane/4 + {0, 8} of a fragment times `scale`, as bf16 at dst + row * ss; rows >= L are not stored.
__device__ __forceinline__ void store_frag_bf16(bf16* dst, long long ss, int row0, int L, const float (&f)[8][4], float scale) {
  const int lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row0 + g + r * 8;
    if (row < L) {
      bf16* d = dst + static_cast<long long>(row) * ss;
#pragma unroll
      for (int t = 0; t < 8; ++t)
        *reinterpret_cast<uint32_t*>(d + t * 8 + 2 * c) = pack_bf16x2(f[t][2 * r] * scale, f[t][2 * r + 1] * scale);
    }
  }
}

// Batch b's bit matrix and tile flags: p.mask / p.tile_flags, or (PER_SEQ) the stack entry mask_index[b] selects.
template <bool PER_SEQ>
__device__ __forceinline__ void batch_mask(const AttnParams& p, int b, const uint32_t*& mask, const uint8_t*& tile_flags) {
  mask = p.mask;
  tile_flags = p.tile_flags;
  if constexpr (PER_SEQ) {
    const long long mi = __ldg(p.mask_index + b);
    mask += mi * p.mask_stride;
    tile_flags += mi * p.flags_stride;
  }
}

// ===================================================== forward ====================================================
template <bool PER_SEQ>
__global__ void __launch_bounds__(128) attn_fwd_kernel(const AttnParams p) {
  __shared__ __align__(1024) uint8_t sm[5 * 8192];
  const uint32_t sQ = smem_u32(sm), sK0 = sQ + 8192, sV0 = sQ + 2 * 8192, sK1 = sQ + 3 * 8192, sV1 = sQ + 4 * 8192;
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
  const int q0 = qt * 64;
  const bf16* qg = p.q + b * p.q_sb + h * p.q_sh;
  const bf16* kg = p.k + b * p.k_sb + h * p.k_sh;
  const bf16* vg = p.v + b * p.v_sb + h * p.v_sh;
  const uint32_t* mask;
  const uint8_t* tile_flags;
  batch_mask<PER_SEQ>(p, b, mask, tile_flags);
  const uint8_t* flags = tile_flags ? tile_flags + static_cast<long long>(qt) * p.nkt : nullptr;

  auto next_tile = [&](int kt) {
    while (kt < p.nkt && flags && flags[kt] == 0) ++kt;
    return kt;
  };

  float o[8][4];
  zero_c(o);
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const float sc = p.scale * LOG2E;
  const long long bh = static_cast<long long>(b) * p.H + h;

  int kt = next_tile(0);
  load_tile_async(sQ, qg, p.q_ss, q0, p.Lq);
  if (kt < p.nkt) {
    load_tile_async(sK0, kg, p.k_ss, kt * 64, p.Lk);
    load_tile_async(sV0, vg, p.v_ss, kt * 64, p.Lk);
  }
  cp_async_commit();
  uint32_t qf[4][4];
  bool q_loaded = false;
  int buf = 0;
  while (kt < p.nkt) {
    const int kt_next = next_tile(kt + 1);
    if (kt_next < p.nkt) {
      load_tile_async(buf ? sK0 : sK1, kg, p.k_ss, kt_next * 64, p.Lk);
      load_tile_async(buf ? sV0 : sV1, vg, p.v_ss, kt_next * 64, p.Lk);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (!q_loaded) { load_a_frags(sQ, warp * 16, qf); q_loaded = true; }
    const uint32_t sK = buf ? sK1 : sK0, sV = buf ? sV1 : sV0;

    float s[8][4];
    zero_c(s);
    mma_a_tT(s, qf, sK);
    fwd_tile_step(p, PER_SEQ ? mask : p.mask, sc, bh, q0 + warp * 16, kt * 64, flags ? flags[kt] : 2, s, o, m_run, l_run);
    uint32_t pa[4][4];
    c_to_a(s, pa);
    mma_p_t(o, pa, sV);
    __syncthreads();
    kt = kt_next;
    buf ^= 1;
  }
  cp_async_wait<0>();

  // ---- finalize (repeated in attn_fwd_wgmma_kernel: as a shared helper it cost this kernel a register) ----
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const float l = quad_sum(l_run[r]);
    const float inv = l > 0.f ? 1.0f / l : 0.f;
    const int row = q0 + warp * 16 + g + r * 8;
    if (row < p.Lq) {
      bf16* dst = p.out + b * p.o_sb + static_cast<long long>(row) * p.o_ss + h * p.o_sh;
#pragma unroll
      for (int t = 0; t < 8; ++t)
        *reinterpret_cast<uint32_t*>(dst + t * 8 + 2 * c) = pack_bf16x2(o[t][2 * r] * inv, o[t][2 * r + 1] * inv);
      if (p.lse && c == 0) p.lse[(bh * p.Lq) + row] = (l > 0.f) ? (m_run[r] + log2f(l)) * LN2 : -INFINITY;
    }
  }
}

// ============================================= forward, wgmma + TMA ===============================================
// Warp-specialised forward for sequences of >= 96 queries.  CTA = 288 threads over the q-tiles 2x and 2x+1 (64 queries
// each) of one (b, h):
//   warps 0-3 / 4-7  consumer warpgroup g: S = Q_g K^T (wgmma m64n64k16, both operands from smem), mask / online softmax /
//                    dropout in registers (fwd_tile_step on each warp's part of the accumulator), P -> bf16 register A
//                    operand, O += P V (wgmma, V read MN-major)
//   warp 8           TMA producer (one thread): Q of both tiles once, then K/V tiles of 64 keys through a 3-stage ring
//                    (mbarrier tx); a K/V tile is loaded when either q-tile sees part of it, and both groups release it.
// 4-D tensor maps (d, seq|head, head|seq, batch) address q/k/v in place in the fused QKV buffer; rows past L are zero.
constexpr int WF_STAGES = 3;
constexpr int WF_THREADS = 288;
constexpr int WF_SMEM = 1024 + 2 * 8192 + WF_STAGES * 2 * 8192 + 128;

__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// 64 rows [row0, row0 + 64) of head h, batch b
__device__ __forceinline__ void tma_rows(uint32_t dst, const CUtensorMap* m, uint64_t* bar, int head_inner, int row0, int h, int b) {
  if (head_inner) tma_load_4d(dst, m, bar, 0, h, row0, b);
  else            tma_load_4d(dst, m, bar, 0, row0, h, b);
}

struct WgmmaFwdMaps { CUtensorMap q, k, v; int q_head_inner, k_head_inner, v_head_inner; };

template <bool PER_SEQ>
__global__ void __launch_bounds__(WF_THREADS, 2) attn_fwd_wgmma_kernel(const __grid_constant__ WgmmaFwdMaps tm, const AttnParams p) {
  extern __shared__ uint8_t wf_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(wf_smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sQ = smem_u32(smem);                       // [2][64 x 128 B]
  const uint32_t sKV = sQ + 2 * 8192;                       // [stage][K 8 KB | V 8 KB]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 2 * 8192 + WF_STAGES * 2 * 8192);
  uint64_t* q_full = bars;
  uint64_t* full = bars + 1;
  uint64_t* empty = full + WF_STAGES;
  const int h = blockIdx.x, b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // late query blocks see the most keys under block-causal masks; blockIdx.z is the slowest launch dimension, so every
  // (b, h) starts its heavy blocks before any light one
  const int qt_base = 2 * (static_cast<int>(gridDim.z) - 1 - static_cast<int>(blockIdx.z));
  const uint32_t* mask;
  const uint8_t* tile_flags;
  batch_mask<PER_SEQ>(p, b, mask, tile_flags);
  const uint8_t* fl0 = tile_flags ? tile_flags + static_cast<long long>(qt_base) * p.nkt : nullptr;
  const bool has1 = qt_base + 1 < p.nqt;
  auto needed = [&](int kt, int g) -> bool {   // does q-tile qt_base+g see any key of k-tile kt?
    if (g == 1 && !has1) return false;
    return !fl0 || fl0[g * p.nkt + kt] != 0;
  };
  auto next_tile = [&](int kt) {
    while (kt < p.nkt && !needed(kt, 0) && !needed(kt, 1)) ++kt;
    return kt;
  };

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int st = 0; st < WF_STAGES; ++st) { mbar_init(&full[st], 1); mbar_init(&empty[st], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ------------------------------------------------ TMA producer ------------------------------------------------
    if (lane == 0) {
      tma_prefetch_desc(&tm.q); tma_prefetch_desc(&tm.k); tma_prefetch_desc(&tm.v);
      mbar_expect_tx(q_full, 2 * 8192);
      tma_rows(sQ, &tm.q, q_full, tm.q_head_inner, qt_base * 64, h, b);
      tma_rows(sQ + 8192, &tm.q, q_full, tm.q_head_inner, qt_base * 64 + 64, h, b);   // past Lq: zero rows
      int st = 0; uint32_t ph = 0;
      for (int kt = next_tile(0); kt < p.nkt; kt = next_tile(kt + 1)) {
        mbar_wait<false>(&empty[st], ph ^ 1);
        mbar_expect_tx(&full[st], 2 * 8192);
        tma_rows(sKV + st * 16384, &tm.k, &full[st], tm.k_head_inner, kt * 64, h, b);
        tma_rows(sKV + st * 16384 + 8192, &tm.v, &full[st], tm.v_head_inner, kt * 64, h, b);
        if (++st == WF_STAGES) { st = 0; ph ^= 1; }
      }
    }
    return;
  }

  // -------------------------------------------------- consumers ---------------------------------------------------
  const int g = warp >> 2, wq = warp & 3;         // consumer group (q-tile qt_base + g), warp within the group
  const int qt = qt_base + g, q0 = qt * 64;
  const uint8_t* flags = fl0 ? fl0 + g * p.nkt : nullptr;
  const long long bh = static_cast<long long>(b) * p.H + h;
  const float sc = p.scale * LOG2E;
  float o[8][4];
  zero_c(o);
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  mbar_wait<false>(q_full, 0);
  const uint32_t qa = sQ + g * 8192;

  int st = 0; uint32_t ph = 0;
  for (int kt = next_tile(0); kt < p.nkt; kt = next_tile(kt + 1)) {
    mbar_wait<false>(&full[st], ph);
    const int flag = flags ? flags[kt] : 2;
    if (flag != 0 && (g == 0 || has1)) {
      const uint32_t ka = sKV + st * 16384, va = ka + 8192;
      float s[8][4];
      float (&sd)[32] = *reinterpret_cast<float(*)[32]>(&s[0][0]);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_m64n64k16_ss(sd, make_smem_desc_sw128(qa + k * 32, 16, 1024), make_smem_desc_sw128(ka + k * 32, 16, 1024), k != 0);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operand32(sd);
      fwd_tile_step(p, PER_SEQ ? mask : p.mask, sc, bh, q0 + wq * 16, kt * 64, flag, s, o, m_run, l_run);
      uint32_t pa[4][4];
      c_to_a(s, pa);
      float (&od)[32] = *reinterpret_cast<float(*)[32]>(&o[0][0]);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_m64n64k16_rs_tb(od, pa[kk], make_smem_desc_sw128(va + kk * 2048, 8192, 1024));
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operand32(od);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[st]);
    if (++st == WF_STAGES) { st = 0; ph ^= 1; }
  }
  if (g == 1 && !has1) return;

  // ---- finalize, as attn_fwd_kernel ----
  const int c = lane & 3, gr = lane >> 2;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const float l = quad_sum(l_run[r]);
    const float inv = l > 0.f ? 1.0f / l : 0.f;
    const int row = q0 + wq * 16 + gr + r * 8;
    if (row < p.Lq) {
      bf16* dst = p.out + b * p.o_sb + static_cast<long long>(row) * p.o_ss + h * p.o_sh;
#pragma unroll
      for (int t = 0; t < 8; ++t)
        *reinterpret_cast<uint32_t*>(dst + t * 8 + 2 * c) = pack_bf16x2(o[t][2 * r] * inv, o[t][2 * r + 1] * inv);
      if (p.lse && c == 0) p.lse[(bh * p.Lq) + row] = (l > 0.f) ? (m_run[r] + log2f(l)) * LN2 : -INFINITY;
    }
  }
}

// ===================================================== delta ======================================================
__global__ void __launch_bounds__(256) attn_delta_kernel(const AttnParams p) {
  // 8 lanes per (b, h, i) row of 64 elements
  const long long idx = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 3;
  const int sub = threadIdx.x & 7;
  const long long total = static_cast<long long>(p.B) * p.H * p.Lq;
  float acc = 0.f;
  if (idx < total) {
    const int i = static_cast<int>(idx % p.Lq);
    const int h = static_cast<int>((idx / p.Lq) % p.H);
    const int b = static_cast<int>(idx / (static_cast<long long>(p.Lq) * p.H));
    const uint4 ou = *reinterpret_cast<const uint4*>(p.o + b * p.o_sb + static_cast<long long>(i) * p.o_ss + h * p.o_sh + sub * 8);
    const uint4 du = *reinterpret_cast<const uint4*>(p.d_o + b * p.do_sb + static_cast<long long>(i) * p.do_ss + h * p.do_sh + sub * 8);
    float2 a, d;
    a = unpack_bf16x2(ou.x); d = unpack_bf16x2(du.x); acc += a.x * d.x + a.y * d.y;
    a = unpack_bf16x2(ou.y); d = unpack_bf16x2(du.y); acc += a.x * d.x + a.y * d.y;
    a = unpack_bf16x2(ou.z); d = unpack_bf16x2(du.z); acc += a.x * d.x + a.y * d.y;
    a = unpack_bf16x2(ou.w); d = unpack_bf16x2(du.w); acc += a.x * d.x + a.y * d.y;
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  acc += __shfl_xor_sync(0xffffffffu, acc, 4);
  if (idx < total && sub == 0) p.delta[idx] = acc;  // layout [B, H, Lq] == idx ordering (b, h, i)? see dispatch
}

// ===================================================== dK / dV ====================================================
// One CTA per (key tile, h, b); warp w owns keys [k0 + 16w, k0 + 16w + 16).  Works on S^T = K Q^T (rows = keys).
__global__ void __launch_bounds__(128) attn_bwd_dkv_kernel(const AttnParams p) {
  __shared__ __align__(1024) uint8_t sm[4 * 8192];
  __shared__ float s_lse[64], s_delta[64];
  __shared__ uint32_t s_mask[64][2];
  const uint32_t sK = smem_u32(sm), sV = sK + 8192, sQ = sK + 2 * 8192, sDO = sK + 3 * 8192;
  const int kt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
  const int k0 = kt * 64;
  const bf16* qg = p.q + b * p.q_sb + h * p.q_sh;
  const bf16* kg = p.k + b * p.k_sb + h * p.k_sh;
  const bf16* vg = p.v + b * p.v_sb + h * p.v_sh;
  const bf16* dog = p.d_o + b * p.do_sb + h * p.do_sh;
  const long long bh = static_cast<long long>(b) * p.H + h;
  const float sc = p.scale * LOG2E;

  load_tile_async(sK, kg, p.k_ss, k0, p.Lk);
  load_tile_async(sV, vg, p.v_ss, k0, p.Lk);
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();
  uint32_t kf[4][4], vf[4][4];
  load_a_frags(sK, warp * 16, kf);
  load_a_frags(sV, warp * 16, vf);

  float dk[8][4], dv[8][4];
  zero_c(dk);
  zero_c(dv);

  for (int qt = 0; qt < p.nqt; ++qt) {
    const int flag = p.tile_flags ? p.tile_flags[static_cast<long long>(qt) * p.nkt + kt] : 2;
    if (flag == 0) continue;
    const int q0 = qt * 64;
    __syncthreads();  // previous iteration's readers are done with sQ / sDO / s_*
    load_tile_async(sQ, qg, p.q_ss, q0, p.Lq);
    load_tile_async(sDO, dog, p.do_ss, q0, p.Lq);
    cp_async_commit();
    if (threadIdx.x < 64) {
      const int qi = q0 + threadIdx.x;
      s_lse[threadIdx.x] = (qi < p.Lq) ? p.lse[bh * p.Lq + qi] * LOG2E : INFINITY;  // +inf => p = 0 for padded rows
      s_delta[threadIdx.x] = (qi < p.Lq) ? p.delta[bh * p.Lq + qi] : 0.f;
      if (flag == 1) {
#pragma unroll
        for (int ww = 0; ww < 2; ++ww) {
          const int wi = kt * 2 + ww;
          s_mask[threadIdx.x][ww] = (qi < p.Lq && wi < p.mask_words) ? p.mask[static_cast<long long>(qi) * p.mask_words + wi] : 0u;
        }
      }
    }
    cp_async_wait<0>();
    __syncthreads();

    // S^T[16 keys x 64 q] = K_w Q^T
    float st[8][4];
    zero_c(st);
    mma_a_tT(st, kf, sQ);
    // dP^T[16 keys x 64 q] = V_w dO^T
    float dpt[8][4];
    zero_c(dpt);
    mma_a_tT(dpt, vf, sDO);

    uint32_t keep[8];
    if (p.drop_scale != 0.f) dropout_bits(p, bh, k0 + warp * 16, q0, true, keep);

    float pt[8][4];
#pragma unroll
    for (int t = 0; t < 8; ++t) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int kr = warp * 16 + g + (e >> 1) * 8;      // key row within tile
        const int qc = t * 8 + 2 * c + (e & 1);           // query col within tile
        bool vis = (k0 + kr < p.Lk);
        if (flag == 1) vis = vis && ((s_mask[qc][kr >> 5] >> (kr & 31)) & 1u);
        const float pv = vis ? exp2f(st[t][e] * sc - s_lse[qc]) : 0.f;
        float dpv = dpt[t][e];
        float pdrop = pv;
        if (p.drop_scale != 0.f) {
          const bool kp = (keep[t] >> e) & 1u;
          pdrop = kp ? pv * p.drop_scale : 0.f;
          dpv = kp ? dpv * p.drop_scale : 0.f;
        }
        pt[t][e] = pdrop;                                  // for dV
        st[t][e] = pv * (dpv - s_delta[qc]);               // dS^T
      }
    }
    uint32_t pa[4][4];
    c_to_a(pt, pa);
    mma_p_t(dv, pa, sDO);   // dV[16 keys x 64 hd] += P^T[16 x 64 q] * dO[64 q x 64 hd]
    c_to_a(st, pa);
    mma_p_t(dk, pa, sQ);    // dK += dS^T * Q
  }
  store_frag_bf16(p.dk + b * p.dk_sb + h * p.dk_sh, p.dk_ss, k0 + warp * 16, p.Lk, dk, p.scale);
  store_frag_bf16(p.dv + b * p.dv_sb + h * p.dv_sh, p.dv_ss, k0 + warp * 16, p.Lk, dv, 1.f);
}

// ===================================================== dQ =========================================================
__global__ void __launch_bounds__(128) attn_bwd_dq_kernel(const AttnParams p) {
  __shared__ __align__(1024) uint8_t sm[4 * 8192];
  const uint32_t sQ = smem_u32(sm), sDO = sQ + 8192, sK = sQ + 2 * 8192, sV = sQ + 3 * 8192;
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5;
  const int q0 = qt * 64;
  const bf16* qg = p.q + b * p.q_sb + h * p.q_sh;
  const bf16* kg = p.k + b * p.k_sb + h * p.k_sh;
  const bf16* vg = p.v + b * p.v_sb + h * p.v_sh;
  const bf16* dog = p.d_o + b * p.do_sb + h * p.do_sh;
  const long long bh = static_cast<long long>(b) * p.H + h;
  const float sc = p.scale * LOG2E;
  const uint8_t* flags = p.tile_flags ? p.tile_flags + static_cast<long long>(qt) * p.nkt : nullptr;

  load_tile_async(sQ, qg, p.q_ss, q0, p.Lq);
  load_tile_async(sDO, dog, p.do_ss, q0, p.Lq);
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();
  uint32_t qf[4][4], dof[4][4];
  load_a_frags(sQ, warp * 16, qf);
  load_a_frags(sDO, warp * 16, dof);
  float lse2[2], dlt[2];
  row_lse_delta(p, bh, q0 + warp * 16, lse2, dlt);
  float dq[8][4];
  zero_c(dq);

  for (int kt = 0; kt < p.nkt; ++kt) {
    const int flag = flags ? flags[kt] : 2;
    if (flag == 0) continue;
    const int k0 = kt * 64;
    __syncthreads();
    load_tile_async(sK, kg, p.k_ss, k0, p.Lk);
    load_tile_async(sV, vg, p.v_ss, k0, p.Lk);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();

    float s[8][4];
    zero_c(s);
    mma_a_tT(s, qf, sK);       // S = Q K^T
    float dp[8][4];
    zero_c(dp);
    mma_a_tT(dp, dof, sV);     // dP = dO V^T
    dq_form_ds(p, sc, bh, q0 + warp * 16, k0, flag, lse2, dlt, s, dp);
    uint32_t pa[4][4];
    c_to_a(s, pa);
    mma_p_t(dq, pa, sK);       // dQ += dS K
  }
  store_frag_bf16(p.dq + b * p.dq_sb + h * p.dq_sh, p.dq_ss, q0 + warp * 16, p.Lq, dq, p.scale);
}

// ============================================ backward, wgmma + TMA ================================================
// Warp-specialised backward for sequences of >= 96 on both sides, in the S^T / dP^T formulation of attn_bwd_dkv_kernel and
// the S / dP one of attn_bwd_dq_kernel (dq_form_ds):
//   DKV = true : unit = key tiles 2z, 2z+1 of one (b, h); consumer group g owns key tile 2z+g (K, V loaded once) and
//                streams query tiles (Q, dO): S^T = K Q^T, dP^T = V dO^T (wgmma, smem x smem), dV += P^T dO,
//                dK += dS^T Q (wgmma, register A operand, Q / dO read MN-major)
//   DKV = false: unit = query tiles 2z, 2z+1; group g owns query tile 2z+g (Q, dO) and streams key tiles (K, V):
//                S = Q K^T, dP = dO V^T, dQ += dS K
// The grid is persistent: CTA c runs units c, c + grid, c + 2 grid, ... (wb_unit gives their order).  Warpgroup 2 is the
// producer: it loads each unit's fixed tiles into one of two buffers and streams the unit's tile pairs through a 3-stage
// ring that carries on across units, so the next unit's fixed tiles and first streamed stages arrive while the consumers
// finish the current one and store its gradients.  A streamed tile is loaded when either group sees it; its thread 0
// issues the TMA loads.  In the dK/dV kernel all 128 of its threads also fill the stage's row statistics (below) before
// they arrive on the stage's full barrier, so the consumers read each query's lse, delta, mask word and dropout keep bits
// with one shared load per two queries instead of per element.  setmaxnreg hands the producer's registers to the
// consumers, which hold dK, dV, S^T and dP^T (128 x 64 + 256 x 216 registers within the 384 x 168 of the launch; at 56
// the producer's Philox draws spill beside the unit it walks).  The consumers issue each k-step of the dV / dK / dQ
// MMAs as soon as its 16 columns of P and dS are formed, so those MMAs run under the rest of the element-wise pass.
struct WgmmaBwdMaps { CUtensorMap f0, f1, s0, s1; int f0_hi, f1_hi, s0_hi, s1_hi; };
constexpr int WB_THREADS = 384;
// Row statistics of one stage's query tile, in 32-bit words: lse * log2(e) and delta of its 64 queries (+inf and 0 past
// Lq), then per consumer group g and mask word ww of its key tile the words [g][ww][query] of the bit mask and of the
// dropout keep bits.  Keep word ww of a query packs its 8-key Philox blocks 4 ww .. 4 ww + 3, the forward's blocks, so
// bit (key & 31) of word key / 32 is the key's keep bit, as in the mask.
constexpr int WB_STAT_LSE = 0, WB_STAT_DELTA = 64, WB_STAT_MASK = 128, WB_STAT_KEEP = 384, WB_STAT_WORDS = 640;
constexpr int WB_FIXED_BYTES = 4 * 8192;                  // one unit's fixed tiles: [group][f0 8 KB | f1 8 KB]

// Unit u = (z * B + b) * H + h: fixed tile pair z of (b, h).  Every (b, h) runs its heaviest pair before any lighter one
// across the whole grid: under block-causal masks early key tiles are seen by the most queries and late query tiles see
// the most keys, so z counts up from the first key pair (dK/dV) or down from the last query pair (dQ).
struct WbUnit { int b, h, ft_base; };
__host__ __device__ inline WbUnit wb_unit(bool dkv, int u, int B, int H, int nf) {
  const int nfb = (nf + 1) / 2;
  const int h = u % H, r = u / H, b = r % B, z = r / B;
  return {b, h, 2 * (dkv ? z : nfb - 1 - z)};
}

template <bool DKV>
// One CTA per SM: dK and dV accumulators next to S and dP need ~160 registers.
__global__ void __launch_bounds__(WB_THREADS, 1) attn_bwd_wgmma_kernel(const __grid_constant__ WgmmaBwdMaps tm, const AttnParams p) {
  extern __shared__ uint8_t wb_smem_raw[];
  // offset from the __shared__ array itself, so that the compiler sees shared-memory accesses (LDS / STS, not generic)
  uint8_t* smem = wb_smem_raw + ((1024 - (smem_u32(wb_smem_raw) & 1023)) & 1023);
  const uint32_t sF = smem_u32(smem);                       // [buffer][group][f0 8 KB | f1 8 KB]
  const uint32_t sS = sF + 2 * WB_FIXED_BYTES;              // [stage][s0 8 KB | s1 8 KB]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 2 * WB_FIXED_BYTES + WF_STAGES * 2 * 8192);
  uint64_t* f_full = bars;                                  // [buffer]
  uint64_t* f_empty = bars + 2;                             // [buffer]
  uint64_t* full = bars + 4;
  uint64_t* empty = full + WF_STAGES;
  uint32_t* stats = reinterpret_cast<uint32_t*>(smem + 2 * WB_FIXED_BYTES + WF_STAGES * 2 * 8192 + 128);   // [stage][WB_STAT_WORDS]
  const int nf = DKV ? p.nkt : p.nqt;                       // tiles on the fixed side
  const int ns = DKV ? p.nqt : p.nkt;                       // tiles on the streamed side
  const int units = (nf + 1) / 2 * p.B * p.H;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int h = 0, b = 0, ft_base = 0;                            // the current unit
  bool has1 = false;
  int bh = 0;                                               // b * H + h
  auto set_unit = [&](int u) {
    const WbUnit w = wb_unit(DKV, u, p.B, p.H, nf);
    h = w.h; b = w.b; ft_base = w.ft_base;
    has1 = ft_base + 1 < nf;
    bh = b * p.H + h;
  };
  auto flag_of = [&](int st_, int g) -> int {               // tile flag of (fixed tile ft_base+g, streamed tile st_)
    if (g == 1 && !has1) return 0;
    if (!p.tile_flags) return 2;
    const int ft = ft_base + g;
    return DKV ? p.tile_flags[static_cast<long long>(st_) * p.nkt + ft] : p.tile_flags[static_cast<long long>(ft) * p.nkt + st_];
  };
  auto next_tile = [&](int t) {
    while (t < ns && flag_of(t, 0) == 0 && flag_of(t, 1) == 0) ++t;
    return t;
  };

  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) { mbar_init(&f_full[i], 1); mbar_init(&f_empty[i], 8); }
    // dK/dV: the TMA thread's expect_tx arrival and one arrival per producer thread once its statistics are written
    for (int st = 0; st < WF_STAGES; ++st) { mbar_init(&full[st], DKV ? 1 + 128 : 1); mbar_init(&empty[st], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 8) {
    setmaxnreg_dec<64>();
    const int pt = threadIdx.x - 256;
    if (!DKV && pt != 0) return;
    if (pt == 0) { tma_prefetch_desc(&tm.f0); tma_prefetch_desc(&tm.f1); tma_prefetch_desc(&tm.s0); tma_prefetch_desc(&tm.s1); }
    const uint64_t seed = p.drop_seed + (p.drop_seed_ptr ? __ldg(p.drop_seed_ptr) : 0ull);
    const int nblk = (p.Lk + 7) >> 3;
    int st = 0; uint32_t ph = 0;
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
      set_unit(u);
      if (pt == 0) {                                        // fixed buffer i % 2, free once unit i - 2 is done with it
        const int i = (u - blockIdx.x) / gridDim.x;         // the CTA's unit count, not carried: the producer's
        const int fb = i & 1;                               // registers are tight around the Philox draws
        mbar_wait<false>(&f_empty[fb], ((i >> 1) & 1) ^ 1);
        mbar_expect_tx(&f_full[fb], WB_FIXED_BYTES);
        const uint32_t dst = sF + fb * WB_FIXED_BYTES;
        for (int g = 0; g < 2; ++g) {                       // a tile past the sequence end is zero-filled
          tma_rows(dst + g * 16384, &tm.f0, &f_full[fb], tm.f0_hi, (ft_base + g) * 64, h, b);
          tma_rows(dst + g * 16384 + 8192, &tm.f1, &f_full[fb], tm.f1_hi, (ft_base + g) * 64, h, b);
        }
      }
      for (int t = next_tile(0); t < ns; t = next_tile(t + 1)) {
        mbar_wait<false>(&empty[st], ph ^ 1);
        if (pt == 0) {
          mbar_expect_tx(&full[st], 2 * 8192);
          tma_rows(sS + st * 16384, &tm.s0, &full[st], tm.s0_hi, t * 64, h, b);
          tma_rows(sS + st * 16384 + 8192, &tm.s1, &full[st], tm.s1_hi, t * 64, h, b);
        }
        if (DKV) {
          // thread pt: lse (pt < 64) or delta (pt >= 64) of query pt % 64; mask and keep words of query pt % 64 for
          // consumer group pt / 64, written only where that group reads them (flag 1 / flag != 0 with dropout)
          uint32_t* sw = stats + st * WB_STAT_WORDS;
          const int qc = pt & 63, gg = pt >> 6;
          const int qi = t * 64 + qc;
          const bool qin = qi < p.Lq;
          if (pt < 64) reinterpret_cast<float*>(sw)[WB_STAT_LSE + qc] = qin ? p.lse[static_cast<long long>(bh) * p.Lq + qi] * LOG2E : INFINITY;
          else         reinterpret_cast<float*>(sw)[WB_STAT_DELTA + qc] = qin ? p.delta[static_cast<long long>(bh) * p.Lq + qi] : 0.f;
          const int flag = flag_of(t, gg);
          const int kb0 = (ft_base + gg) * 8;               // first 8-key block of the group's key tile
#pragma unroll
          for (int ww = 0; ww < 2; ++ww) {
            const int slot = (gg * 2 + ww) * 64 + qc;
            if (flag == 1) {
              const int wi = (kb0 >> 2) + ww;
              sw[WB_STAT_MASK + slot] = (qin && wi < p.mask_words) ? __ldg(p.mask + static_cast<long long>(qi) * p.mask_words + wi) : 0u;
            }
            if (flag != 0 && p.drop_scale != 0.f) {
              uint32_t kw = 0;
#pragma unroll
              for (int j = 0; j < 4; ++j)
                kw |= dropout_keep8(seed, (static_cast<long long>(bh) * p.Lq + qi) * nblk + kb0 + ww * 4 + j, p.drop_thresh) << (8 * j);
              sw[WB_STAT_KEEP + slot] = kw;
            }
          }
          mbar_arrive(&full[st]);
        }
        if (++st == WF_STAGES) { st = 0; ph ^= 1; }
      }
    }
    return;
  }

  setmaxnreg_inc<216>();
  const int g = warp >> 2, wq = warp & 3;
  const int c = lane & 3, gr = lane >> 2;
  const float sc = p.scale * LOG2E;
  int st = 0; uint32_t ph = 0;
  for (int u = blockIdx.x, i = 0; u < units; u += gridDim.x, ++i) {
    set_unit(u);
    const int fb = i & 1;
    const int f0 = (ft_base + g) * 64;                      // first key (DKV) / query (dQ) row of this group
    const uint32_t fa0 = sF + fb * WB_FIXED_BYTES + g * 16384, fa1 = fa0 + 8192;   // DKV: K, V of the key tile; dQ: Q, dO
    float acc0[8][4], acc1[8][4];                           // DKV: dK, dV; dQ: dQ (acc1 unused)
    zero_c(acc0);
    zero_c(acc1);
    float lse2[2], dlt[2];
    if (!DKV) row_lse_delta(p, bh, f0 + wq * 16, lse2, dlt);
    mbar_wait<false>(&f_full[fb], (i >> 1) & 1);

    for (int t = next_tile(0); t < ns; t = next_tile(t + 1)) {
      mbar_wait<false>(&full[st], ph);
      const int flag = flag_of(t, g);
      const uint32_t sa0 = sS + st * 16384, sa1 = sa0 + 8192;   // DKV: Q, dO of the query tile; dQ: K, V of the key tile
      float s[8][4], dp[8][4];
      float (&sd)[32] = *reinterpret_cast<float(*)[32]>(&s[0][0]);
      float (&dpd)[32] = *reinterpret_cast<float(*)[32]>(&dp[0][0]);
      if (flag != 0) {
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_m64n64k16_ss(sd, make_smem_desc_sw128(fa0 + k * 32, 16, 1024), make_smem_desc_sw128(sa0 + k * 32, 16, 1024), k != 0);
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_m64n64k16_ss(dpd, make_smem_desc_sw128(fa1 + k * 32, 16, 1024), make_smem_desc_sw128(sa1 + k * 32, 16, 1024), k != 0);
        wgmma_commit();
        const int s0r = t * 64;
        wgmma_wait<0>();
        wgmma_fence_operand32(sd);
        wgmma_fence_operand32(dpd);
        if (DKV) {
          // ---- as attn_bwd_dkv_kernel: rows = keys (f0 + ...), cols = queries (s0r + ...), with the query's lse, delta,
          // mask word and keep bits from the stage's statistics (the producer wrote them before the full barrier) ----
          const int k0 = f0;
          const uint32_t* sw = stats + st * WB_STAT_WORDS;
          const int slot = (g * 2 + (wq >> 1)) * 64;            // mask / keep word of this warp's 16 key rows
          float pt[8][4];
          uint32_t pa[4][4], da[4][4];
          float (&dkd)[32] = *reinterpret_cast<float(*)[32]>(&acc0[0][0]);
          float (&dvd)[32] = *reinterpret_cast<float(*)[32]>(&acc1[0][0]);
          // 16 queries at a time: their P^T and dS^T columns are the A operand of k-step kk of dV += P^T dO and
          // dK += dS^T Q, issued as soon as they are formed so the MMAs run under the next columns' element-wise pass.
          // Each accumulator still takes its k-steps in order.
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
            for (int tt = 2 * kk; tt < 2 * kk + 2; ++tt) {
              const int qc = tt * 8 + 2 * c;                    // this thread's queries qc, qc + 1 of the tile
              const float2 lse_q = *reinterpret_cast<const float2*>(sw + WB_STAT_LSE + qc);
              const float2 dlt_q = *reinterpret_cast<const float2*>(sw + WB_STAT_DELTA + qc);
              uint2 mw = make_uint2(~0u, ~0u), kw = make_uint2(0u, 0u);   // mask words: all ones outside partial tiles
              if (flag == 1) mw = *reinterpret_cast<const uint2*>(sw + WB_STAT_MASK + slot + qc);
              if (p.drop_scale != 0.f) kw = *reinterpret_cast<const uint2*>(sw + WB_STAT_KEEP + slot + qc);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const int kr = wq * 16 + gr + (e >> 1) * 8;
                const float lse_e = (e & 1) ? lse_q.y : lse_q.x, dlt_e = (e & 1) ? dlt_q.y : dlt_q.x;
                // a hidden key's exponent is -inf, so P is +0 without a branch
                const bool vis = (k0 + kr < p.Lk) && ((((e & 1) ? mw.y : mw.x) >> (kr & 31)) & 1u);
                const float pv = exp2f(vis ? s[tt][e] * sc - lse_e : -INFINITY);
                float dpv = dp[tt][e];
                float pdrop = pv;
                if (p.drop_scale != 0.f) {
                  const bool kp = ((((e & 1) ? kw.y : kw.x) >> (kr & 31)) & 1u);
                  pdrop = kp ? pv * p.drop_scale : 0.f;
                  dpv = kp ? dpv * p.drop_scale : 0.f;
                }
                pt[tt][e] = pdrop;
                s[tt][e] = pv * (dpv - dlt_e);
              }
            }
            pa[kk][0] = pack_bf16x2(pt[2 * kk][0], pt[2 * kk][1]);       // c_to_a, k-step kk
            pa[kk][1] = pack_bf16x2(pt[2 * kk][2], pt[2 * kk][3]);
            pa[kk][2] = pack_bf16x2(pt[2 * kk + 1][0], pt[2 * kk + 1][1]);
            pa[kk][3] = pack_bf16x2(pt[2 * kk + 1][2], pt[2 * kk + 1][3]);
            da[kk][0] = pack_bf16x2(s[2 * kk][0], s[2 * kk][1]);
            da[kk][1] = pack_bf16x2(s[2 * kk][2], s[2 * kk][3]);
            da[kk][2] = pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
            da[kk][3] = pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
            wgmma_fence();
            wgmma_m64n64k16_rs_tb(dvd, pa[kk], make_smem_desc_sw128(sa1 + kk * 2048, 8192, 1024));
            wgmma_m64n64k16_rs_tb(dkd, da[kk], make_smem_desc_sw128(sa0 + kk * 2048, 8192, 1024));
          }
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_operand32(dkd);
          wgmma_fence_operand32(dvd);
        } else {
          // rows = queries (f0 + ...), cols = keys (s0r + ...); k-step kk of dQ += dS K is issued once dS has its 16 keys,
          // as in the dK/dV kernel
          DqTileBits tb;
          dq_tile_bits(p, bh, f0 + wq * 16, s0r, flag, tb);
          uint32_t da[4][4];
          float (&dqd)[32] = *reinterpret_cast<float(*)[32]>(&acc0[0][0]);
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            dq_ds_cols(p, sc, s0r, lse2, dlt, tb, s, dp, 2 * kk, 2 * kk + 2);
            da[kk][0] = pack_bf16x2(s[2 * kk][0], s[2 * kk][1]);        // c_to_a, k-step kk
            da[kk][1] = pack_bf16x2(s[2 * kk][2], s[2 * kk][3]);
            da[kk][2] = pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
            da[kk][3] = pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
            wgmma_fence();
            wgmma_m64n64k16_rs_tb(dqd, da[kk], make_smem_desc_sw128(sa0 + kk * 2048, 8192, 1024));
          }
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_operand32(dqd);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[st]);
      if (++st == WF_STAGES) { st = 0; ph ^= 1; }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&f_empty[fb]);               // the fixed tiles are read by the S/dP MMAs only
    if (g == 1 && !has1) continue;
    if (DKV) {
      store_frag_bf16(p.dk + b * p.dk_sb + h * p.dk_sh, p.dk_ss, f0 + wq * 16, p.Lk, acc0, p.scale);
      store_frag_bf16(p.dv + b * p.dv_sb + h * p.dv_sh, p.dv_ss, f0 + wq * 16, p.Lk, acc1, 1.f);
    } else {
      store_frag_bf16(p.dq + b * p.dq_sb + h * p.dq_sh, p.dq_ss, f0 + wq * 16, p.Lq, acc0, p.scale);
    }
  }
}
constexpr int WB_SMEM = 1024 + 2 * WB_FIXED_BYTES + WF_STAGES * 2 * 8192 + 128 + WF_STAGES * WB_STAT_WORDS * 4;

// ===================================================== mask tiles =================================================
__global__ void attn_mask_tiles_kernel(const uint32_t* __restrict__ mask, int mask_words, int Lq, int Lk, int nkt,
                                       uint8_t* __restrict__ flags) {
  // one warp per (qt, kt)
  const int tile = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int nqt = (Lq + 63) / 64;
  if (tile >= nqt * nkt) return;
  const int qt = tile / nkt, kt = tile % nkt;
  int any = 0, all = 1;
  for (int i = lane; i < 128; i += 32) {  // 64 rows x 2 words
    const int row = qt * 64 + (i >> 1), wi = kt * 2 + (i & 1);
    if (row >= Lq) continue;
    const int kbase = wi * 32;
    if (kbase >= Lk) continue;
    const uint32_t valid = (Lk - kbase >= 32) ? 0xffffffffu : ((1u << (Lk - kbase)) - 1u);
    const uint32_t w = (wi < mask_words ? mask[static_cast<long long>(row) * mask_words + wi] : 0u) & valid;
    any |= (w != 0u);
    all &= (w == valid);
  }
  any = __any_sync(0xffffffffu, any);
  all = __all_sync(0xffffffffu, all);
  if (lane == 0) flags[tile] = any ? (all ? 2 : 1) : 0;
}

// ============================================ observation-token drop ==============================================
// The pretrain phase's per-forward mask (dreamvla_model.py:55-59): for every timestep i, `count` of its n_obs observation
// columns are hidden from that timestep's action rows.  Column j of timestep i draws the key r(i, j) =
// philox4x32(seed + *seed_ptr, i * n_obs + j).x; the `count` columns with the smallest (r, j) are dropped -- a uniform
// count-subset per timestep, independent across timesteps.  One block per timestep: rank every key against the others in
// shared memory, then write the timestep's rows of `bits` = `base` with the dropped (action row, obs column) bits cleared.
constexpr int OBS_DROP_THREADS = 256;
constexpr int OBS_DROP_MAX_OBS = OBS_DROP_THREADS;

__global__ void __launch_bounds__(OBS_DROP_THREADS)
attn_mask_obs_drop_kernel(const uint32_t* __restrict__ base, uint32_t* __restrict__ bits, int mask_words, int n_tok,
                          int num_A, int n_obs, int n_act, int count, uint64_t seed, const int64_t* __restrict__ seed_ptr) {
  __shared__ uint64_t key[OBS_DROP_MAX_OBS];
  __shared__ uint32_t span[OBS_DROP_MAX_OBS / 32 + 1];   // drop bits of the obs columns, aligned to the mask's words
  const int i = blockIdx.x, t = threadIdx.x;
  const uint64_t eff = seed + (seed_ptr ? static_cast<uint64_t>(*seed_ptr) : 0ull);
  const int c0 = i * n_tok + num_A;                      // first observation column of timestep i
  const int w0 = c0 >> 5, w1 = (c0 + n_obs - 1) >> 5;    // the words those columns span (n_obs >= 1)
  if (t < n_obs) {
    const uint32_t r = philox4x32(eff, static_cast<uint64_t>(i) * n_obs + t).x;
    key[t] = (static_cast<uint64_t>(r) << 32) | static_cast<uint32_t>(t);   // distinct keys: ties broken by j
  }
  if (t <= w1 - w0) span[t] = 0u;
  __syncthreads();
  if (t < n_obs) {
    const uint64_t mine = key[t];
    int rank = 0;
    for (int k = 0; k < n_obs; ++k) rank += key[k] < mine;
    if (rank < count) atomicOr(&span[((c0 + t) >> 5) - w0], 1u << ((c0 + t) & 31));
  }
  __syncthreads();
  const int a0 = num_A + n_obs;                          // first action row of the timestep, relative to its first row
  const long long row0 = static_cast<long long>(i) * n_tok;
  for (int e = t; e < n_tok * mask_words; e += OBS_DROP_THREADS) {
    const int rr = e / mask_words, w = e - rr * mask_words;
    uint32_t v = base[(row0 + rr) * mask_words + w];
    if (rr >= a0 && rr < a0 + n_act && w >= w0 && w <= w1) v &= ~span[w - w0];
    bits[(row0 + rr) * mask_words + w] = v;
  }
}

// ===================================================== host =======================================================
static bool strides_ok(const void* ptr, long long sb, long long ss, long long sh) {
  return ptr && aligned16(ptr) && sb % 8 == 0 && ss % 8 == 0 && sh % 8 == 0;
}

bool attn_small_applicable(int64_t Lq, int64_t Lk, const void* mask, float dropout_p);   // attention_small.cu
int attn_small_fwd(const dvla_attn_fwd_args* a, cudaStream_t s);
int attn_small_bwd(const dvla_attn_bwd_args* a, cudaStream_t s);

// head_dim 0 (callers built before the field existed) and 64 run on every kernel; 96 only on the short-sequence ones.
static bool head_dim_ok(int64_t head_dim, bool small) { return head_dim == 0 || head_dim == 64 || (head_dim == 96 && small); }
template <class Args>
static int head_dim_unsupported(const char* op, const Args* a) {
  set_error("%s: head_dim %lld unsupported: 64, or 96 on the short-sequence kernels only (Lq <= 32, Lk <= 64, no mask, "
            "no dropout); got Lq=%lld Lk=%lld mask=%s dropout_p=%g", op, (long long)a->head_dim, (long long)a->Lq,
            (long long)a->Lk, a->mask ? "yes" : "no", (double)a->dropout_p);
  return DVLA_ERR_UNSUPPORTED;
}

// [B, L, H, 64] strided view -> 4-D tensor map with 64 x 64 boxes, 128-byte swizzle (the layout the wgmma descriptors
// expect); seq and head dims are ordered so that the strides ascend.
static bool make_attn_tmap(CUtensorMap* out, const void* base, long long L, long long H, long long B, long long ss,
                           long long sh, long long sb, int* head_inner) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point not found"); return false; }
  *head_inner = (sh <= ss) ? 1 : 0;
  cuuint64_t dims[4]; cuuint64_t strides[3]; cuuint32_t box[4]; cuuint32_t estr[4] = {1, 1, 1, 1};
  dims[0] = 64; box[0] = 64;
  if (*head_inner) { dims[1] = H; dims[2] = L; strides[0] = sh * 2; strides[1] = ss * 2; box[1] = 1; box[2] = 64; }
  else             { dims[1] = L; dims[2] = H; strides[0] = ss * 2; strides[1] = sh * 2; box[1] = 64; box[2] = 1; }
  dims[3] = B; box[3] = 1;
  strides[2] = (B > 1 ? sb : (long long)dims[1] * dims[2] * 64) * 2;
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("attn tensor map encode failed (%d): L=%lld H=%lld B=%lld ss=%lld sh=%lld sb=%lld", (int)r, L, H, B, ss, sh, sb);
    return false;
  }
  return true;
}

// Strides a tensor map can express: positive, distinct seq / head strides, a head's rows not overlapping the next head.
static bool tmap_strides_ok(long long L, long long H, long long B, long long ss, long long sh, long long sb) {
  if (ss <= 0 || sh <= 0 || ss == sh || (B > 1 && sb <= 0)) return false;
  return (sh < ss) ? (sh >= 64 && ss >= sh * H) : (ss >= 64 && sh >= ss * L);
}

template <bool PER_SEQ>
static int attn_fwd_wgmma_launch(const dvla_attn_fwd_args* a, const AttnParams& p, cudaStream_t s) {
  WgmmaFwdMaps tm;
  if (!make_attn_tmap(&tm.q, a->q, a->Lq, a->H, a->B, a->q_ss, a->q_sh, a->q_sb, &tm.q_head_inner) ||
      !make_attn_tmap(&tm.k, a->k, a->Lk, a->H, a->B, a->k_ss, a->k_sh, a->k_sb, &tm.k_head_inner) ||
      !make_attn_tmap(&tm.v, a->v, a->Lk, a->H, a->B, a->v_ss, a->v_sh, a->v_sb, &tm.v_head_inner))
    return DVLA_ERR_CUDA;
  static std::once_flag once;
  static cudaError_t attr_err = cudaSuccess;
  if (!set_smem_attr_once(once, attr_err, attn_fwd_wgmma_kernel<PER_SEQ>, WF_SMEM)) { set_error("attn_fwd_wgmma smem attribute: %s", cudaGetErrorString(attr_err)); return DVLA_ERR_CUDA; }
  attn_fwd_wgmma_kernel<PER_SEQ><<<dim3(p.H, p.B, (p.nqt + 1) / 2), WF_THREADS, WF_SMEM, s>>>(tm, p);
  DVLA_CHECK_LAUNCH("attn_fwd_wgmma");
  return DVLA_OK;
}

template <bool DKV>
static int attn_bwd_wgmma_launch(const WgmmaBwdMaps& tm, const AttnParams& p, cudaStream_t s) {
  static std::once_flag once;
  static cudaError_t attr_err = cudaSuccess;
  if (!set_smem_attr_once(once, attr_err, attn_bwd_wgmma_kernel<DKV>, WB_SMEM)) { set_error("attn_bwd_wgmma smem attribute: %s", cudaGetErrorString(attr_err)); return DVLA_ERR_CUDA; }
  const int nf = DKV ? p.nkt : p.nqt;
  const long long units = (long long)(nf + 1) / 2 * p.B * p.H;
  if (units > INT_MAX) { set_error("attn_bwd_wgmma: %lld work units exceed the int index", units); return DVLA_ERR_UNSUPPORTED; }
  const int grid = units < num_sms() ? (int)units : num_sms();   // persistent: one CTA per SM the budget leaves us
  attn_bwd_wgmma_kernel<DKV><<<grid, WB_THREADS, WB_SMEM, s>>>(tm, p);
  DVLA_CHECK_LAUNCH(DKV ? "attn_bwd_dkv_wgmma" : "attn_bwd_dq_wgmma");
  return DVLA_OK;
}

// The AttnParams fields the forward and backward share: operands q/k/v, o and lse, dims, tile counts, mask and dropout.
template <class Args>
static AttnParams attn_params(const Args* a) {
  AttnParams p;
  memset(&p, 0, sizeof(p));
  p.q = (const bf16*)a->q; p.k = (const bf16*)a->k; p.v = (const bf16*)a->v; p.lse = const_cast<float*>(a->lse);
  p.mask = a->mask; p.tile_flags = a->mask ? a->tile_flags : nullptr;
  p.B = (int)a->B; p.H = (int)a->H; p.Lq = (int)a->Lq; p.Lk = (int)a->Lk;
  p.nqt = (p.Lq + 63) / 64; p.nkt = (p.Lk + 63) / 64; p.mask_words = a->mask_words;
  p.q_sb = a->q_sb; p.q_ss = a->q_ss; p.q_sh = a->q_sh; p.k_sb = a->k_sb; p.k_ss = a->k_ss; p.k_sh = a->k_sh;
  p.v_sb = a->v_sb; p.v_ss = a->v_ss; p.v_sh = a->v_sh; p.o_sb = a->o_sb; p.o_ss = a->o_ss; p.o_sh = a->o_sh;
  p.scale = a->scale;
  if (a->dropout_p > 0.f) {
    dropout_thresh_scale(a->dropout_p, &p.drop_thresh, &p.drop_scale);
    p.drop_seed = a->dropout_seed;
    p.drop_seed_ptr = a->dropout_seed_ptr;
  }
  return p;
}

}  // namespace dvla

using namespace dvla;

extern "C" int dvla_attn_fwd(const dvla_attn_fwd_args* a, void* stream) {
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!a) { set_error("attn_fwd: null args"); return DVLA_ERR_INVALID; }
  if (!strides_ok(a->q, a->q_sb, a->q_ss, a->q_sh) || !strides_ok(a->k, a->k_sb, a->k_ss, a->k_sh) ||
      !strides_ok(a->v, a->v_sb, a->v_ss, a->v_sh) || !strides_ok(a->o, a->o_sb, a->o_ss, a->o_sh)) {
    set_error("attn_fwd: q/k/v/o must be non-null, 16-byte aligned with strides multiple of 8 elements");
    return DVLA_ERR_INVALID;
  }
  if (a->B <= 0 || a->H <= 0 || a->Lq <= 0 || a->Lk <= 0) { set_error("attn_fwd: non-positive dims"); return DVLA_ERR_INVALID; }
  if (a->H > 65535 || a->B > 65535) { set_error("attn_fwd: B,H must be <= 65535"); return DVLA_ERR_UNSUPPORTED; }
  if (a->mask && a->mask_words * 32 < a->Lk) { set_error("attn_fwd: mask_words too small"); return DVLA_ERR_INVALID; }
  if (a->mask && !a->tile_flags) { set_error("attn_fwd: mask given without tile_flags"); return DVLA_ERR_INVALID; }
  if (!dropout_rate_ok(a->dropout_p)) { set_error("attn_fwd: dropout_p out of range [0, 1)"); return DVLA_ERR_INVALID; }
  const bool small = attn_small_applicable(a->Lq, a->Lk, a->mask, a->dropout_p);
  if (!head_dim_ok(a->head_dim, small)) return head_dim_unsupported("attn_fwd", a);
  // (the short-sequence kernels take no mask, so there a mask_index always lacks one)
  const bool index_without_mask = a->mask_index && !a->mask;
  if (small && !index_without_mask) return attn_small_fwd(a, s);
  if (a->key_bias && !small) {
    set_error("attn_fwd: key_bias needs the short-sequence kernels (Lq <= 32, Lk <= 64, no mask, no dropout)");
    return DVLA_ERR_UNSUPPORTED;
  }
  if (index_without_mask) { set_error("attn_fwd: mask_index given without mask"); return DVLA_ERR_INVALID; }
  if (a->mask_index && (a->mask_stride < 0 || a->flags_stride < 0)) {
    set_error("attn_fwd: negative mask_stride %lld / flags_stride %lld", (long long)a->mask_stride, (long long)a->flags_stride);
    return DVLA_ERR_INVALID;
  }
  AttnParams p = attn_params(a);
  p.out = (bf16*)a->o;
  // a mask implies the kernels below (the short-sequence ones take none), and each has a per-sequence-mask variant
  const bool per_seq = a->mask_index != nullptr;
  p.mask_index = a->mask_index; p.mask_stride = a->mask_stride; p.flags_stride = a->flags_stride;
  // wgmma + TMA for the long sequences (backbone, ViT, decoders); the mma.sync kernel for short query blocks and strides a
  // tensor map cannot express
  if (a->Lq >= 96 && tmap_strides_ok(a->Lq, a->H, a->B, a->q_ss, a->q_sh, a->q_sb) &&
      tmap_strides_ok(a->Lk, a->H, a->B, a->k_ss, a->k_sh, a->k_sb) && tmap_strides_ok(a->Lk, a->H, a->B, a->v_ss, a->v_sh, a->v_sb))
    return per_seq ? attn_fwd_wgmma_launch<true>(a, p, s) : attn_fwd_wgmma_launch<false>(a, p, s);
  if (per_seq) attn_fwd_kernel<true><<<dim3(p.nqt, p.H, p.B), 128, 0, s>>>(p);
  else         attn_fwd_kernel<false><<<dim3(p.nqt, p.H, p.B), 128, 0, s>>>(p);
  DVLA_CHECK_LAUNCH("attn_fwd");
  return DVLA_OK;
}

extern "C" int dvla_attn_bwd(const dvla_attn_bwd_args* a, void* stream) {
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!a) { set_error("attn_bwd: null args"); return DVLA_ERR_INVALID; }
  if (!strides_ok(a->q, a->q_sb, a->q_ss, a->q_sh) || !strides_ok(a->k, a->k_sb, a->k_ss, a->k_sh) ||
      !strides_ok(a->v, a->v_sb, a->v_ss, a->v_sh) || !strides_ok(a->o, a->o_sb, a->o_ss, a->o_sh) ||
      !strides_ok(a->d_o, a->do_sb, a->do_ss, a->do_sh) || !strides_ok(a->dq, a->dq_sb, a->dq_ss, a->dq_sh) ||
      !strides_ok(a->dk, a->dk_sb, a->dk_ss, a->dk_sh) || !strides_ok(a->dv, a->dv_sb, a->dv_ss, a->dv_sh)) {
    set_error("attn_bwd: tensors must be non-null, 16-byte aligned with strides multiple of 8 elements");
    return DVLA_ERR_INVALID;
  }
  if (!a->lse || !a->delta) { set_error("attn_bwd: lse/delta null"); return DVLA_ERR_INVALID; }
  if (a->B <= 0 || a->H <= 0 || a->Lq <= 0 || a->Lk <= 0) { set_error("attn_bwd: non-positive dims"); return DVLA_ERR_INVALID; }
  if (a->mask && !a->tile_flags) { set_error("attn_bwd: mask given without tile_flags"); return DVLA_ERR_INVALID; }
  if (!dropout_rate_ok(a->dropout_p)) { set_error("attn_bwd: dropout_p out of range [0, 1)"); return DVLA_ERR_INVALID; }
  const bool small = attn_small_applicable(a->Lq, a->Lk, a->mask, a->dropout_p);
  if (!head_dim_ok(a->head_dim, small)) return head_dim_unsupported("attn_bwd", a);
  if (small) return attn_small_bwd(a, s);   // writes delta itself
  if (a->key_bias) {
    set_error("attn_bwd: key_bias needs the short-sequence kernels (Lq <= 32, Lk <= 64, no mask, no dropout)");
    return DVLA_ERR_UNSUPPORTED;
  }
  AttnParams p = attn_params(a);
  p.o = (const bf16*)a->o; p.d_o = (const bf16*)a->d_o; p.dq = (bf16*)a->dq; p.dk = (bf16*)a->dk; p.dv = (bf16*)a->dv;
  p.delta = a->delta;
  p.do_sb = a->do_sb; p.do_ss = a->do_ss; p.do_sh = a->do_sh;
  p.dq_sb = a->dq_sb; p.dq_ss = a->dq_ss; p.dq_sh = a->dq_sh; p.dk_sb = a->dk_sb; p.dk_ss = a->dk_ss; p.dk_sh = a->dk_sh;
  p.dv_sb = a->dv_sb; p.dv_ss = a->dv_ss; p.dv_sh = a->dv_sh;
  const long long rows = (long long)p.B * p.H * p.Lq;
  attn_delta_kernel<<<(unsigned)((rows * 8 + 255) / 256), 256, 0, s>>>(p);
  DVLA_CHECK_LAUNCH("attn_delta");
  // wgmma + TMA when both sequences are long and every operand is tensor-map addressable; mma.sync kernels otherwise
  if (a->Lq >= 96 && a->Lk >= 96 && a->B <= 65535 && a->H <= 65535 &&
      tmap_strides_ok(a->Lq, a->H, a->B, a->q_ss, a->q_sh, a->q_sb) && tmap_strides_ok(a->Lq, a->H, a->B, a->do_ss, a->do_sh, a->do_sb) &&
      tmap_strides_ok(a->Lk, a->H, a->B, a->k_ss, a->k_sh, a->k_sb) && tmap_strides_ok(a->Lk, a->H, a->B, a->v_ss, a->v_sh, a->v_sb)) {
    CUtensorMap tq, tdo, tk, tv;
    int hq, hdo, hk, hv;
    if (!make_attn_tmap(&tq, a->q, a->Lq, a->H, a->B, a->q_ss, a->q_sh, a->q_sb, &hq) ||
        !make_attn_tmap(&tdo, a->d_o, a->Lq, a->H, a->B, a->do_ss, a->do_sh, a->do_sb, &hdo) ||
        !make_attn_tmap(&tk, a->k, a->Lk, a->H, a->B, a->k_ss, a->k_sh, a->k_sb, &hk) ||
        !make_attn_tmap(&tv, a->v, a->Lk, a->H, a->B, a->v_ss, a->v_sh, a->v_sb, &hv))
      return DVLA_ERR_CUDA;
    const WgmmaBwdMaps dkv{tk, tv, tq, tdo, hk, hv, hq, hdo};
    const WgmmaBwdMaps dq{tq, tdo, tk, tv, hq, hdo, hk, hv};
    const int rc = attn_bwd_wgmma_launch<true>(dkv, p, s);
    if (rc != DVLA_OK) return rc;
    return attn_bwd_wgmma_launch<false>(dq, p, s);
  }
  attn_bwd_dkv_kernel<<<dim3(p.nkt, p.H, p.B), 128, 0, s>>>(p);
  DVLA_CHECK_LAUNCH("attn_bwd_dkv");
  attn_bwd_dq_kernel<<<dim3(p.nqt, p.H, p.B), 128, 0, s>>>(p);
  DVLA_CHECK_LAUNCH("attn_bwd_dq");
  return DVLA_OK;
}

extern "C" int dvla_attn_mask_tiles(const uint32_t* mask, int32_t mask_words, int64_t Lq, int64_t Lk, uint8_t* flags,
                                    void* stream) {
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!mask || !flags) { set_error("attn_mask_tiles: null pointer"); return DVLA_ERR_INVALID; }
  if (mask_words * 32 < Lk) { set_error("attn_mask_tiles: mask_words too small"); return DVLA_ERR_INVALID; }
  const int nqt = (int)((Lq + 63) / 64), nkt = (int)((Lk + 63) / 64);
  const int tiles = nqt * nkt;
  attn_mask_tiles_kernel<<<(tiles + 3) / 4, 128, 0, s>>>(mask, mask_words, (int)Lq, (int)Lk, nkt, flags);
  DVLA_CHECK_LAUNCH("attn_mask_tiles");
  return DVLA_OK;
}

extern "C" int dvla_attn_mask_obs_drop(const uint32_t* base_bits, uint32_t* bits, uint8_t* tile_flags, int32_t mask_words,
                                       int64_t L, int64_t K, int64_t n_tok, int64_t num_A, int64_t n_obs, int64_t n_act,
                                       int64_t count, uint64_t seed, const int64_t* seed_ptr, void* stream) {
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!base_bits || !bits || !tile_flags) { set_error("attn_mask_obs_drop: null pointer"); return DVLA_ERR_INVALID; }
  if (base_bits == bits) { set_error("attn_mask_obs_drop: bits must not alias base_bits"); return DVLA_ERR_INVALID; }
  if (L <= 0 || L > (1 << 24) || mask_words <= 0 || static_cast<int64_t>(mask_words) * 32 < L) {
    set_error("attn_mask_obs_drop: L=%lld with mask_words=%d (need 0 < L <= 32 * mask_words)", (long long)L, (int)mask_words);
    return DVLA_ERR_INVALID;
  }
  if (K <= 0 || n_tok <= 0 || K * n_tok != L) {
    set_error("attn_mask_obs_drop: layout K=%lld x n_tok=%lld does not tile L=%lld", (long long)K, (long long)n_tok, (long long)L);
    return DVLA_ERR_INVALID;
  }
  if (num_A < 0 || n_obs < 1 || n_act < 0 || num_A + n_obs + n_act > n_tok) {
    set_error("attn_mask_obs_drop: num_A=%lld + n_obs=%lld + n_act=%lld outside n_tok=%lld (n_obs >= 1)", (long long)num_A,
              (long long)n_obs, (long long)n_act, (long long)n_tok);
    return DVLA_ERR_INVALID;
  }
  if (n_obs > OBS_DROP_MAX_OBS) {
    set_error("attn_mask_obs_drop: n_obs=%lld above the kernel's limit of %d", (long long)n_obs, OBS_DROP_MAX_OBS);
    return DVLA_ERR_INVALID;
  }
  if (count < 0 || count > n_obs) {
    set_error("attn_mask_obs_drop: count=%lld outside [0, n_obs=%lld]", (long long)count, (long long)n_obs);
    return DVLA_ERR_INVALID;
  }
  attn_mask_obs_drop_kernel<<<(unsigned)K, OBS_DROP_THREADS, 0, s>>>(base_bits, bits, mask_words, (int)n_tok, (int)num_A,
                                                                     (int)n_obs, (int)n_act, (int)count, seed, seed_ptr);
  DVLA_CHECK_LAUNCH("attn_mask_obs_drop");
  return dvla_attn_mask_tiles(bits, mask_words, L, L, tile_flags, stream);
}

extern "C" int64_t dvla_attn_bwd_workspace_bytes(int64_t B, int64_t H, int64_t Lq) {
  return (B > 0 && H > 0 && Lq > 0) ? 4 * B * H * Lq : 0;
}
