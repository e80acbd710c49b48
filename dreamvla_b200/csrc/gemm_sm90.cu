// Persistent, warp-specialised wgmma GEMM with fused epilogue for sm_90a.
//
//   out[M,N] = epi(alpha * A[M,K] * B[N,K]^T)          bf16 operands, fp32 accumulation in registers
//
// CTA = 384 threads (3 warpgroups), one CTA per SM (persistent over work units, static round-robin), 128 x 128 tiles:
//   warpgroup 0     TMA producer (one thread): cp.async.bulk.tensor -> 128B-swizzled smem ring (4 stages), mbarrier tx
//   warpgroups 1-2  consumers: wgmma.mma_async m64n128k16 on rows [64*g, 64*g+64) of the tile, accumulators in
//                   registers; a stage is handed back to the producer once the wgmma group that read it has retired.
//                   After the last k-block each consumer writes its accumulators to an fp32 smem tile, and its 4 warps
//                   run the fused epilogue (bias/act/dact/dropout/residual) on 32 x 32 chunks, one row per lane.
// While the consumers run an epilogue the producer is already filling the ring with the next unit's k-blocks.
// Both operands may be K-major or MN-major (wgmma transpose bits), which covers forward, dgrad and wgrad for nn.Linear
// ([out,in]) and HF Conv1D ([in,out]) weights without any transpose pass.
//
// Replaces the cuBLAS calls behind nn.Linear / Conv1D in the reference (see include/dvla.h for call sites).
#include "common.cuh"
#include "host.cuh"
#include "../../include/dvla.h"

namespace dvla {

constexpr int BM = 128;
constexpr int BN = 128;
constexpr int BK = 64;       // 64 bf16 = 128 B = one swizzle row
constexpr int WG_K = 16;     // k of one wgmma
constexpr int NUM_CONSUMERS = 2;                       // consumer warpgroups, 64 rows each
constexpr int NUM_EPI_WARPS = 4 * NUM_CONSUMERS;
constexpr int EPI_STAGE_BYTES = 2048;  // per epilogue warp: 32 rows x 64 B staging panel
constexpr int GEMM_THREADS = 128 * (1 + NUM_CONSUMERS);
constexpr int ACC_LD = BN + 4;         // fp32 row stride of the accumulator tile in smem (+4: conflict-free row reads)

struct GemmParams {
  void* out;
  const bf16* bias;
  const void* residual;
  bf16* aux_out;
  const bf16* aux_in;
  int M, N, K;
  long long ldo, ldr, ld_aux;
  int num_m_tiles, num_n_tiles, num_k_blocks;
  int act, out_fp32, vec_ok, staged_ok;
  int k_splits, kb_per_split;   // split-K: work unit = (tile, split), each covering kb_per_split k-blocks
  int atomic_out;               // epilogue = out += v with red.global.add.bf16x2 (split-K accumulate into a gradient)
  // K-split TAIL (see map_unit): tiles [tail_first, total) are each cut into tail_splits k-ranges of tail_kbps k-blocks; the
  // partial accumulators meet in an fp32 workspace and the LAST unit to arrive runs the normal epilogue on the full sum
  int tail_first, tail_splits, tail_kbps;
  float* tail_ws;               // [CTA slot][8 warp regions][split][chunk][8][32 lanes][4] fp32 partial accumulators
  unsigned* tail_cnt;           // [CTA slot][8] arrival counters, all zero between launches
  float alpha;
  float drop_scale;        // 1/(1-p_eff), 0 => dropout disabled
  uint32_t drop_thresh;    // round(p*65536)
  uint64_t drop_seed;
  const uint64_t* drop_seed_ptr;
};

struct GemmCfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = 4;
  static constexpr int ACC_BYTES = BM * ACC_LD * 4;
  static constexpr int BAR_BYTES = 256;
  static constexpr int STAGING_BYTES = NUM_EPI_WARPS * EPI_STAGE_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + ACC_BYTES + STAGING_BYTES + 1024 + BAR_BYTES;
};
static_assert(GemmCfg::SMEM_BYTES <= 227 * 1024, "GEMM shared memory exceeds the sm_90 per-block limit");

// ---- epilogue for 8 consecutive columns of one row ---------------------------------------------------------------
__device__ __forceinline__ void epilogue8(float (&v)[8], int row, int col, const GemmParams& p) {
  const bool full = p.vec_ok && (col + 8 <= p.N);
  const int nvalid = min(8, p.N - col);
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] *= p.alpha;
  if (p.bias) {
    if (full) {
      uint4 b = __ldg(reinterpret_cast<const uint4*>(p.bias + col));
      float2 f;
      f = unpack_bf16x2(b.x); v[0] += f.x; v[1] += f.y;
      f = unpack_bf16x2(b.y); v[2] += f.x; v[3] += f.y;
      f = unpack_bf16x2(b.z); v[4] += f.x; v[5] += f.y;
      f = unpack_bf16x2(b.w); v[6] += f.x; v[7] += f.y;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (j < nvalid) v[j] += __bfloat162float(p.bias[col + j]);
    }
  }
  if (p.aux_out) {
    bf16* dst = p.aux_out + static_cast<long long>(row) * p.ld_aux + col;
    if (full) {
      uint4 o = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]),
                           pack_bf16x2(v[6], v[7]));
      *reinterpret_cast<uint4*>(dst) = o;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (j < nvalid) dst[j] = __float2bfloat16(v[j]);
    }
  }
  if (p.aux_in) {
    const bf16* src = p.aux_in + static_cast<long long>(row) * p.ld_aux + col;
    float x[8];
    if (full) {
      uint4 a = __ldg(reinterpret_cast<const uint4*>(src));
      float2 f;
      f = unpack_bf16x2(a.x); x[0] = f.x; x[1] = f.y;
      f = unpack_bf16x2(a.y); x[2] = f.x; x[3] = f.y;
      f = unpack_bf16x2(a.z); x[4] = f.x; x[5] = f.y;
      f = unpack_bf16x2(a.w); x[6] = f.x; x[7] = f.y;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) x[j] = (j < nvalid) ? __bfloat162float(src[j]) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] *= act_bwd(x[j], p.act);
  } else if (p.act != ACT_NONE) {
    act_fwd_n<8>(v, p.act);
  }
  if (p.drop_scale != 0.f) {
    // RNG block = row*ceil(N/8) + col/8, bit col%8 (include/dvla.h; the same mask as dvla_dropout): each row starts a new
    // block, so the mask of an element depends on its (row, col) only, never on the tiling.
    const uint64_t blk = static_cast<uint64_t>(row) * static_cast<uint64_t>((p.N + 7) >> 3) + (col >> 3);
    const uint64_t seed = p.drop_seed + (p.drop_seed_ptr ? __ldg(p.drop_seed_ptr) : 0ull);
    const uint32_t keep = dropout_keep8(seed, blk, p.drop_thresh);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = ((keep >> j) & 1u) ? v[j] * p.drop_scale : 0.f;
  }
  if (p.out_fp32) {
    float* dst = reinterpret_cast<float*>(p.out) + static_cast<long long>(row) * p.ldo + col;
    if (p.residual) {
      const float* r = reinterpret_cast<const float*>(p.residual) + static_cast<long long>(row) * p.ldr + col;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (j < nvalid) v[j] += r[j];
    }
    if (full) {
      reinterpret_cast<float4*>(dst)[0] = make_float4(v[0], v[1], v[2], v[3]);
      reinterpret_cast<float4*>(dst)[1] = make_float4(v[4], v[5], v[6], v[7]);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (j < nvalid) dst[j] = v[j];
    }
  } else {
    bf16* dst = reinterpret_cast<bf16*>(p.out) + static_cast<long long>(row) * p.ldo + col;
    if (p.residual) {
      const bf16* r = reinterpret_cast<const bf16*>(p.residual) + static_cast<long long>(row) * p.ldr + col;
      if (full) {
        uint4 a = *reinterpret_cast<const uint4*>(r);
        float2 f;
        f = unpack_bf16x2(a.x); v[0] += f.x; v[1] += f.y;
        f = unpack_bf16x2(a.y); v[2] += f.x; v[3] += f.y;
        f = unpack_bf16x2(a.z); v[4] += f.x; v[5] += f.y;
        f = unpack_bf16x2(a.w); v[6] += f.x; v[7] += f.y;
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (j < nvalid) v[j] += __bfloat162float(r[j]);
      }
    }
    if (full) {
      uint4 o = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]),
                           pack_bf16x2(v[6], v[7]));
      *reinterpret_cast<uint4*>(dst) = o;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (j < nvalid) dst[j] = __float2bfloat16(v[j]);
    }
  }
}

// ---- staged epilogue: per-warp 32 x 64 B smem panel (32 rows x 32 bf16 columns) ---------------------------------------
// The one-row-per-lane chunk layout gives each lane 32 contiguous bf16 of ONE row; writing those straight to global costs 32 L1
// wavefronts per store instruction.  Staging through this swizzled panel (16-byte chunk c of row r stored at
// c ^ ((r >> 1) & 3): conflict-free for both the row-wise writes and the 8-rows-per-instruction reads) turns every
// global access of the epilogue (output, pre-activation copy, residual) into full 64-byte row segments.
__device__ __forceinline__ uint4* stage_ptr(uint8_t* base, int row, int chunk) {
  return reinterpret_cast<uint4*>(base + row * 64 + ((chunk ^ ((row >> 1) & 3)) << 4));
}
__device__ __forceinline__ void stage_write_row(uint8_t* base, int lane, const float (&v)[32]) {
#pragma unroll
  for (int c = 0; c < 4; ++c)
    *stage_ptr(base, lane, c) = make_uint4(pack_bf16x2(v[8 * c], v[8 * c + 1]), pack_bf16x2(v[8 * c + 2], v[8 * c + 3]),
                                           pack_bf16x2(v[8 * c + 4], v[8 * c + 5]), pack_bf16x2(v[8 * c + 6], v[8 * c + 7]));
}
// panel (rows row0.., cols col0..col0+31) <-> global [*, ld] bf16; rows >= M and 8-col groups >= N are skipped
__device__ __forceinline__ void stage_flush(uint8_t* base, int lane, bf16* g, long long ld, int row0, int col0, int M, int N) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = i * 8 + (lane >> 2), c = lane & 3;
    if (row0 + r < M && col0 + c * 8 < N)
      *reinterpret_cast<uint4*>(g + static_cast<long long>(row0 + r) * ld + col0 + c * 8) = *stage_ptr(base, r, c);
  }
}
// out += panel with one 16-byte vector reduction per 8 columns (REDG.E.ADD.BF16x8)
__device__ __forceinline__ void stage_flush_atomic(uint8_t* base, int lane, bf16* g, long long ld, int row0, int col0, int M, int N) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = i * 8 + (lane >> 2), c = lane & 3;
    if (row0 + r < M && col0 + c * 8 < N) {
      const uint4 v = *stage_ptr(base, r, c);
      asm volatile("red.global.add.noftz.v4.bf16x2 [%0], {%1, %2, %3, %4};"
                   :: "l"(g + static_cast<long long>(row0 + r) * ld + col0 + c * 8), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
                   : "memory");
    }
  }
}
__device__ __forceinline__ void stage_load(uint8_t* base, int lane, const bf16* g, long long ld, int row0, int col0, int M, int N) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = i * 8 + (lane >> 2), c = lane & 3;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (row0 + r < M && col0 + c * 8 < N)
      val = *reinterpret_cast<const uint4*>(g + static_cast<long long>(row0 + r) * ld + col0 + c * 8);
    *stage_ptr(base, r, c) = val;
  }
}

// one 32-column chunk of one warp: v[32] = this lane's row (row0 + lane), columns col0 .. col0+31
__device__ __forceinline__ void epilogue_chunk_staged(float (&v)[32], uint8_t* stage, int lane, int row0, int col0,
                                                      const GemmParams& p) {
  const int row = row0 + lane;
  if (p.alpha != 1.0f) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] *= p.alpha;
  }
  if (p.bias) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      if (col0 + c * 8 < p.N) {
        const uint4 b = __ldg(reinterpret_cast<const uint4*>(p.bias + col0 + c * 8));
        float2 f;
        f = unpack_bf16x2(b.x); v[8 * c] += f.x; v[8 * c + 1] += f.y;
        f = unpack_bf16x2(b.y); v[8 * c + 2] += f.x; v[8 * c + 3] += f.y;
        f = unpack_bf16x2(b.z); v[8 * c + 4] += f.x; v[8 * c + 5] += f.y;
        f = unpack_bf16x2(b.w); v[8 * c + 6] += f.x; v[8 * c + 7] += f.y;
      }
    }
  }
  if (p.aux_out) {
    stage_write_row(stage, lane, v);
    __syncwarp();
    stage_flush(stage, lane, p.aux_out, p.ld_aux, row0, col0, p.M, p.N);
    __syncwarp();
  }
  if (p.aux_in) {
    stage_load(stage, lane, p.aux_in, p.ld_aux, row0, col0, p.M, p.N);
    __syncwarp();
    float x[32];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const uint4 a = *stage_ptr(stage, lane, c);
      float2 f;
      f = unpack_bf16x2(a.x); x[8 * c] = f.x; x[8 * c + 1] = f.y;
      f = unpack_bf16x2(a.y); x[8 * c + 2] = f.x; x[8 * c + 3] = f.y;
      f = unpack_bf16x2(a.z); x[8 * c + 4] = f.x; x[8 * c + 5] = f.y;
      f = unpack_bf16x2(a.w); x[8 * c + 6] = f.x; x[8 * c + 7] = f.y;
    }
    act_bwd_mul_n<32>(v, x, p.act);
    __syncwarp();
  } else if (p.act != ACT_NONE) {
    act_fwd_n<32>(v, p.act);
  }
  if (p.drop_scale != 0.f) {
    const uint64_t seed = p.drop_seed + (p.drop_seed_ptr ? __ldg(p.drop_seed_ptr) : 0ull);
    const uint64_t blk0 = static_cast<uint64_t>(row) * static_cast<uint64_t>((p.N + 7) >> 3) + (col0 >> 3);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const uint32_t keep = dropout_keep8(seed, blk0 + c, p.drop_thresh);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[8 * c + j] = ((keep >> j) & 1u) ? v[8 * c + j] * p.drop_scale : 0.f;
    }
  }
  if (p.residual) {
    stage_load(stage, lane, reinterpret_cast<const bf16*>(p.residual), p.ldr, row0, col0, p.M, p.N);
    __syncwarp();
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const uint4 a = *stage_ptr(stage, lane, c);
      float2 f;
      f = unpack_bf16x2(a.x); v[8 * c] += f.x; v[8 * c + 1] += f.y;
      f = unpack_bf16x2(a.y); v[8 * c + 2] += f.x; v[8 * c + 3] += f.y;
      f = unpack_bf16x2(a.z); v[8 * c + 4] += f.x; v[8 * c + 5] += f.y;
      f = unpack_bf16x2(a.w); v[8 * c + 6] += f.x; v[8 * c + 7] += f.y;
    }
    __syncwarp();
  }
  stage_write_row(stage, lane, v);
  __syncwarp();
  if (p.atomic_out) stage_flush_atomic(stage, lane, reinterpret_cast<bf16*>(p.out), p.ldo, row0, col0, p.M, p.N);
  else              stage_flush(stage, lane, reinterpret_cast<bf16*>(p.out), p.ldo, row0, col0, p.M, p.N);
  __syncwarp();
}

// Accumulator hand-off and epilogue.  Consumer warpgroup g owns rows [64g, 64g+64) of the tile; its fp32 accumulators go
// to acc_tile (row stride ACC_LD), then warp w (0..3) of the group takes column chunk w (32 columns) of both 32-row halves:
// lane l handles row l of a chunk, the layout the staged epilogue below is written for.
constexpr int CPW = 2;   // 32 x 32 chunks per epilogue warp and tile

__device__ __forceinline__ void store_acc_fragment(float* acc_tile, const float (&d)[64], int warp_in_group, int lane) {
  const int r = 16 * warp_in_group + (lane >> 2);
  const int c = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    *reinterpret_cast<float2*>(acc_tile + r * ACC_LD + 8 * j + c) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(acc_tile + (r + 8) * ACC_LD + 8 * j + c) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}
// chunk ci of this warp: row (32*ci + lane) of the group's 64 rows, columns [32*w, 32*w+32)
__device__ __forceinline__ void load_acc_chunk(const float* acc_tile, int warp_in_group, int ci, int lane, float (&v)[32]) {
  const float* src = acc_tile + (32 * ci + lane) * ACC_LD + 32 * warp_in_group;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 t = *reinterpret_cast<const float4*>(src + 4 * j);
    v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
  }
}

// Epilogue of one output tile for one epilogue warp; m0g = first row of the warp's consumer group.
__device__ __forceinline__ void epilogue_tile(const float* acc_tile, uint8_t* stage, int warp_in_group, int lane, int m0g,
                                              int n0, const GemmParams& p) {
  const int c0 = n0 + 32 * warp_in_group;
  if (c0 >= p.N) return;     // warp-uniform
#pragma unroll 1
  for (int ci = 0; ci < CPW; ++ci) {
    const int r0 = m0g + 32 * ci;
    if (r0 >= p.M) break;
    float v[32];
    load_acc_chunk(acc_tile, warp_in_group, ci, lane, v);
    if (p.staged_ok) {
      epilogue_chunk_staged(v, stage, lane, r0, c0, p);
    } else {
      const int row = r0 + lane;
      if (row < p.M) {
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const int col = c0 + g * 8;
          if (col < p.N) {
            float w[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) w[j] = v[g * 8 + j];
            epilogue8(w, row, col, p);
          }
        }
      }
    }
  }
}

// ---- work units ---------------------------------------------------------------------------------------------------
// A persistent CTA (pair) walks units round-robin.  Without a tail: unit = (tile, uniform k-split).  With a tail
// (p.tail_splits > 1): units [0, tail_first) are whole tiles -- a whole number of waves -- and the tiles that would form
// the last, partly filled wave are cut along K so that every CTA (pair) gets ~1/tail_splits of a tile instead of a
// few getting a whole one while the rest idle:  2.2 waves of tiles cost 2.2 tile-times instead of 3.
struct Unit { int tile, kb0, kb1, slot, split; };   // slot < 0: whole tile / atomic split-K; >= 0: tail tile index
__host__ __device__ __forceinline__ int gemm_total_units(int total_tiles, const GemmParams& p) {
  return p.tail_splits > 1 ? p.tail_first + (total_tiles - p.tail_first) * p.tail_splits : total_tiles * p.k_splits;
}
__host__ __device__ __forceinline__ Unit map_unit(int unit, int total_tiles, const GemmParams& p) {
  Unit u;
  if (p.tail_splits > 1) {
    u.split = 0;
    if (unit < p.tail_first) { u.tile = unit; u.kb0 = 0; u.kb1 = p.num_k_blocks; u.slot = -1; return u; }
    const int t = unit - p.tail_first, nt = total_tiles - p.tail_first;
    u.slot = t % nt;
    u.tile = p.tail_first + u.slot;
    u.split = t / nt;
    u.kb0 = u.split * p.tail_kbps;
    u.kb1 = u.kb0 + p.tail_kbps < p.num_k_blocks ? u.kb0 + p.tail_kbps : p.num_k_blocks;
    return u;
  }
  u.tile = unit % total_tiles;
  u.kb0 = (unit / total_tiles) * p.kb_per_split;
  u.kb1 = u.kb0 + p.kb_per_split < p.num_k_blocks ? u.kb0 + p.kb_per_split : p.num_k_blocks;
  u.slot = -1;
  u.split = 0;
  return u;
}

// Epilogue of one K-split tail unit for one epilogue warp.  The warp owns the same 64-row x 32-column region of the tile
// in every split, so the reduction is per warp region, with no CTA-wide synchronisation and no atomics on data:
//   1. smem accumulators -> this split's fp32 slice of the workspace, 16 bytes per lane per store ([chunk][col/4][lane][4]:
//      a warp instruction writes 512 contiguous bytes);
//   2. __threadfence, one atomicAdd on the region's arrival counter;
//   3. the warp that arrives LAST sums the slices of all splits in split order (L2 reads, ld.cg) -- a fixed order, so the
//      result does not depend on which split finished last -- resets the counter, and runs the ordinary fused epilogue
//      (bias / act / dropout / residual / aux) on the sum: one rounding to bf16 whatever the number of splits.
__device__ __forceinline__ void epilogue_tile_tail(const float* acc_tile, uint8_t* stage, int epi_warp, int warp_in_group,
                                                   int lane, int m0g, int n0, const GemmParams& p, int cta_slot, int split) {
  constexpr int REGION = CPW * 32 * 32;                      // floats per warp region
  const long long region = static_cast<long long>(cta_slot) * NUM_EPI_WARPS + epi_warp;
  float* base = p.tail_ws + region * p.tail_splits * REGION + lane * 4;     // + split * REGION + (ci * 8 + j) * 128
  float* mine = base + static_cast<long long>(split) * REGION;
#pragma unroll 1
  for (int ci = 0; ci < CPW; ++ci) {
    float v[32];
    load_acc_chunk(acc_tile, warp_in_group, ci, lane, v);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      __stcg(reinterpret_cast<float4*>(mine + (ci * 8 + j) * 128), make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]));
  }
  __threadfence();
  __syncwarp();
  unsigned arrived = 0;
  if (lane == 0) arrived = atomicAdd(p.tail_cnt + region, 1u);
  arrived = __shfl_sync(0xffffffffu, arrived, 0);
  if (arrived != static_cast<unsigned>(p.tail_splits - 1)) return;
  __threadfence();
  if (lane == 0) p.tail_cnt[region] = 0u;
  const int c0 = n0 + 32 * warp_in_group;
  if (c0 >= p.N) return;     // warp-uniform
#pragma unroll 1
  for (int ci = 0; ci < CPW; ++ci) {
    const int r0 = m0g + 32 * ci;
    if (r0 >= p.M) break;
    float v[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = 0.f;
#pragma unroll 1
    for (int sp = 0; sp < p.tail_splits; ++sp) {
      const float* src = base + static_cast<long long>(sp) * REGION + ci * 8 * 128;
      float4 t[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) t[j] = __ldcg(reinterpret_cast<const float4*>(src + j * 128));
#pragma unroll
      for (int j = 0; j < 8; ++j) { v[4 * j] += t[j].x; v[4 * j + 1] += t[j].y; v[4 * j + 2] += t[j].z; v[4 * j + 3] += t[j].w; }
    }
    epilogue_chunk_staged(v, stage, lane, r0, c0, p);
  }
}

template <bool A_MN, bool B_MN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const GemmParams p) {
  using Cfg = GemmCfg;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + Cfg::STAGES * Cfg::A_BYTES;
  float* acc_smem = reinterpret_cast<float*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES);
  uint8_t* staging = reinterpret_cast<uint8_t*>(acc_smem) + Cfg::ACC_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + Cfg::STAGING_BYTES);
  uint64_t* empty_bar = full_bar + Cfg::STAGES;

  const int wg = threadIdx.x >> 7;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], NUM_EPI_WARPS);    // lane 0 of every consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int total_tiles = p.num_m_tiles * p.num_n_tiles;
  const int total_units = gemm_total_units(total_tiles, p);

  if (wg == 0) {
    // ------------------------------------------------ TMA producer ------------------------------------------------
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int unit = blockIdx.x; unit < total_units; unit += gridDim.x) {
        const Unit u = map_unit(unit, total_tiles, p);
        const int m0 = (u.tile % p.num_m_tiles) * BM;
        const int n0 = (u.tile / p.num_m_tiles) * BN;
        for (int kb = u.kb0; kb < u.kb1; ++kb) {
          mbar_wait<false>(&empty_bar[s], ph ^ 1);
          mbar_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
          uint8_t* a_dst = sA + s * Cfg::A_BYTES;
          uint8_t* b_dst = sB + s * Cfg::B_BYTES;
          if (!A_MN) {
            tma_load_2d(a_dst, &tmA, &full_bar[s], kb * BK, m0);
          } else {
#pragma unroll
            for (int i = 0; i < BM / 64; ++i) tma_load_2d(a_dst + i * (BK * 128), &tmA, &full_bar[s], m0 + i * 64, kb * BK);
          }
          if (!B_MN) {
            tma_load_2d(b_dst, &tmB, &full_bar[s], kb * BK, n0);
          } else {
#pragma unroll
            for (int i = 0; i < BN / 64; ++i) tma_load_2d(b_dst + i * (BK * 128), &tmB, &full_bar[s], n0 + i * 64, kb * BK);
          }
          if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
    return;
  }

  // -------------------------------------------------- consumers ---------------------------------------------------
  setmaxnreg_inc<232>();                     // 128 x 40 + 256 x 232 registers <= 64 K
  const int g = wg - 1;                      // consumer group: rows [64g, 64g+64) of the tile
  const int warp_in_group = warp & 3;
  const int epi_warp = warp - 4;             // 0 .. NUM_EPI_WARPS-1
  float* acc_tile = acc_smem + g * 64 * ACC_LD;
  uint8_t* stage = staging + epi_warp * EPI_STAGE_BYTES;
  float d[64];
  int s = 0;
  uint32_t ph = 0;
  for (int unit = blockIdx.x; unit < total_units; unit += gridDim.x) {
    const Unit u = map_unit(unit, total_tiles, p);
    const int m0 = (u.tile % p.num_m_tiles) * BM;
    const int n0 = (u.tile / p.num_m_tiles) * BN;
    int prev = -1;
    for (int kb = u.kb0; kb < u.kb1; ++kb) {
      mbar_wait<false>(&full_bar[s], ph);
      const uint32_t a_base = smem_u32(sA + s * Cfg::A_BYTES) + g * (64 * 128);   // K-major: 64 rows; MN-major: 64-wide atom g
      const uint32_t b_base = smem_u32(sB + s * Cfg::B_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / WG_K; ++k) {
        const uint64_t a_desc = A_MN ? make_smem_desc_sw128(a_base + k * (WG_K * 128), BK * 128, 1024)
                                     : make_smem_desc_sw128(a_base + k * (WG_K * 2), 16, 1024);
        const uint64_t b_desc = B_MN ? make_smem_desc_sw128(b_base + k * (WG_K * 128), BK * 128, 1024)
                                     : make_smem_desc_sw128(b_base + k * (WG_K * 2), 16, 1024);
        wgmma_m64n128k16_bf16<A_MN ? 1 : 0, B_MN ? 1 : 0>(d, a_desc, b_desc, ((kb - u.kb0) | k) != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<1>();                         // the group that read stage `prev` has retired: hand it back
      wgmma_fence_operand(d);
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      prev = s;
      if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_operand(d);
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
    }
    named_barrier_sync(1 + g, 128);            // the group's previous epilogue has finished reading acc_tile
    store_acc_fragment(acc_tile, d, warp_in_group, lane);
    named_barrier_sync(1 + g, 128);
    if (u.slot >= 0)
      epilogue_tile_tail(acc_tile, stage, epi_warp, warp_in_group, lane, m0 + 64 * g, n0, p, u.slot, u.split);
    else
      epilogue_tile(acc_tile, stage, warp_in_group, lane, m0 + 64 * g, n0, p);
  }
}

// ---- SIMT kernels of identical semantics for operands TMA cannot address (unaligned strides, K or N < 8) -------------
// thread-per-(row, 8 columns) for short contractions; warp-per-(row, 8 columns) with a lane-strided k loop when the
// contraction is long and the output small (wgrad of the 7-wide DiT layers: 5 k outputs x K = 960).
__device__ __forceinline__ float simt_a(const bf16* a, long long lda, int a_mn, int row, int k) {
  return __bfloat162float(a_mn ? a[static_cast<long long>(k) * lda + row] : a[static_cast<long long>(row) * lda + k]);
}
__device__ __forceinline__ float simt_b(const bf16* b, long long ldb, int b_mn, int n, int k) {
  return __bfloat162float(b_mn ? b[static_cast<long long>(k) * ldb + n] : b[static_cast<long long>(n) * ldb + k]);
}
__global__ void gemm_simt_kernel(const bf16* __restrict__ a, const bf16* __restrict__ b, long long lda, long long ldb,
                                 int a_mn, int b_mn, GemmParams p) {
  const long long groups_n = (p.N + 7) / 8;
  const long long gid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= static_cast<long long>(p.M) * groups_n) return;
  const int row = static_cast<int>(gid / groups_n);
  const int col = static_cast<int>(gid % groups_n) * 8;
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = 0.f;
  const int nvalid = min(8, p.N - col);
  for (int k = 0; k < p.K; ++k) {
    const float av = simt_a(a, lda, a_mn, row, k);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (j < nvalid) v[j] = fmaf(av, simt_b(b, ldb, b_mn, col + j, k), v[j]);
  }
  epilogue8(v, row, col, p);
}
__global__ void gemm_simt_warp_kernel(const bf16* __restrict__ a, const bf16* __restrict__ b, long long lda, long long ldb,
                                      int a_mn, int b_mn, GemmParams p) {
  const long long groups_n = (p.N + 7) / 8;
  const long long wid = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= static_cast<long long>(p.M) * groups_n) return;      // warp-uniform
  const int row = static_cast<int>(wid / groups_n);
  const int col = static_cast<int>(wid % groups_n) * 8;
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = 0.f;
  const int nvalid = min(8, p.N - col);
  for (int k = lane; k < p.K; k += 32) {
    const float av = simt_a(a, lda, a_mn, row, k);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (j < nvalid) v[j] = fmaf(av, simt_b(b, ldb, b_mn, col + j, k), v[j]);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = warp_sum(v[j]);
  if (lane == 0) epilogue8(v, row, col, p);
}

}  // namespace dvla

// ============================================== host side ========================================================
#include <mutex>
#include <unordered_map>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

namespace dvla {

// dvla_gemm_plan: the dispatcher runs as usual up to the point where it would encode tensor maps and launch; with this
// thread-local set it records its decisions instead (host only -- no CUDA call, usable without a GPU)
static thread_local dvla_gemm_plan_info* g_plan = nullptr;
static void record_plan(const GemmParams& p, int kernel, int tile_m, int tile_n, int m_tiles, int grid_ctas) {
  dvla_gemm_plan_info& o = *g_plan;
  o.kernel = kernel; o.tile_m = tile_m; o.tile_n = tile_n;
  o.m_tiles = m_tiles; o.n_tiles = p.num_n_tiles; o.k_blocks = p.num_k_blocks;
  o.k_splits = p.k_splits; o.kb_per_split = p.kb_per_split; o.atomic_out = p.atomic_out;
  o.tail_first = p.tail_first; o.tail_splits = p.tail_splits; o.tail_kbps = p.tail_kbps;
  o.units = kernel >= 2 ? gemm_total_units(m_tiles * p.num_n_tiles, p) : 0;
  o.grid_ctas = grid_ctas;
}

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  });
  return fn;
}

// Descriptor cache (SURVEY 8b): the only mutable module-level state besides the launch counter.  Keyed by everything
// cuTensorMapEncodeTiled sees; guarded by a mutex because forward (main thread) and backward (autograd's device thread)
// call into the library concurrently.  Bounded: cleared when full (activations are recycled by the caching allocator, so
// a training loop touches a few thousand distinct (pointer, shape) pairs).
struct TmapKey {
  const void* base; uint64_t inner, outer, ld; uint32_t box_inner, box_outer;
  bool operator==(const TmapKey& o) const {
    return base == o.base && inner == o.inner && outer == o.outer && ld == o.ld && box_inner == o.box_inner && box_outer == o.box_outer;
  }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    uint64_t h = reinterpret_cast<uint64_t>(k.base) * 0x9E3779B97F4A7C15ull;
    h ^= (k.inner + 0x632BE59BD9B4E019ull) * 0xD1342543DE82EF95ull; h = (h << 13) | (h >> 51);
    h ^= (k.outer << 20) ^ (k.ld * 0xA0761D6478BD642Full) ^ ((uint64_t)k.box_inner << 40) ^ ((uint64_t)k.box_outer << 52);
    return static_cast<size_t>(h ^ (h >> 29));
  }
};
static std::mutex g_tmap_mu;
static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> g_tmap_cache;
constexpr size_t TMAP_CACHE_MAX = 8192;

// 2-D bf16 tensor map: inner dim contiguous, 128B swizzle, zero OOB fill.
bool make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer, uint64_t ld_elems,
                       uint32_t box_inner, uint32_t box_outer) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point not found"); return false; }
  const TmapKey key{base, inner, outer, ld_elems, box_inner, box_outer};
  {
    std::lock_guard<std::mutex> lk(g_tmap_mu);
    auto it = g_tmap_cache.find(key);
    if (it != g_tmap_cache.end()) { *out = it->second; return true; }
  }
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld_elems * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): inner=%llu outer=%llu ld=%llu box=%ux%u base=%p", (int)r,
              (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)ld_elems, box_inner, box_outer,
              base);
    return false;
  }
  {
    std::lock_guard<std::mutex> lk(g_tmap_mu);
    if (g_tmap_cache.size() >= TMAP_CACHE_MAX) g_tmap_cache.clear();
    g_tmap_cache.emplace(key, *out);
  }
  return true;
}

template <bool A_MN, bool B_MN>
static int launch_tc(const dvla_gemm_args* a, const GemmParams& p, cudaStream_t stream) {
  using Cfg = GemmCfg;
  const int units = gemm_total_units(p.num_m_tiles * p.num_n_tiles, p);
  const int grid = units < num_sms() ? units : num_sms();
  if (g_plan) {
    record_plan(p, 2, BM, BN, p.num_m_tiles, grid);
    return DVLA_OK;
  }
  CUtensorMap tmA, tmB;
  if (!A_MN) { if (!make_tmap_2d_bf16(&tmA, a->a, a->K, a->M, a->lda, BK, BM)) return DVLA_ERR_CUDA; }
  else       { if (!make_tmap_2d_bf16(&tmA, a->a, a->M, a->K, a->lda, 64, BK)) return DVLA_ERR_CUDA; }
  if (!B_MN) { if (!make_tmap_2d_bf16(&tmB, a->b, a->K, a->N, a->ldb, BK, BN)) return DVLA_ERR_CUDA; }
  else       { if (!make_tmap_2d_bf16(&tmB, a->b, a->N, a->K, a->ldb, 64, BK)) return DVLA_ERR_CUDA; }
  auto kern = gemm_wgmma_kernel<A_MN, B_MN>;
  static std::once_flag once;      // per instantiation
  static cudaError_t attr_err = cudaSuccess;
  if (!set_smem_attr_once(once, attr_err, kern, Cfg::SMEM_BYTES)) {
    set_error("cudaFuncSetAttribute(smem=%d): %s", Cfg::SMEM_BYTES, cudaGetErrorString(attr_err)); return DVLA_ERR_CUDA;
  }
  kern<<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, stream>>>(tmA, tmB, p);
  DVLA_CHECK_LAUNCH("gemm_wgmma");
  return DVLA_OK;
}

static int launch_tc_any(const dvla_gemm_args* a, const GemmParams& p, cudaStream_t stream) {
  switch ((a->a_mn_major ? 2 : 0) | (a->b_mn_major ? 1 : 0)) {
    case 0: return launch_tc<false, false>(a, p, stream);
    case 1: return launch_tc<false, true>(a, p, stream);
    case 2: return launch_tc<true, false>(a, p, stream);
    default: return launch_tc<true, true>(a, p, stream);
  }
}

// DVLA_GEMM_SPLITK=0 disables the atomic split-K path (bit-reproducible gradient accumulation order)
static bool splitk_enabled() {
  static const bool on = [] { const char* e = getenv("DVLA_GEMM_SPLITK"); return !(e && !strcmp(e, "0")); }();
  return on;
}

// workspace = [16384 arrival counters (64 KB), zero between launches] [fp32 partial tiles: 128 x 128 x 4 bytes per CTA and split]
constexpr int64_t TAIL_CNT_BYTES = 65536;
constexpr int64_t TAIL_WS_SLICES = 132;              // 128 x 128 fp32 slices (8.25 MB): a split tail wave needs <= 132 (one
                                                     // per SM)

static bool tail_fits(const dvla_gemm_args* a, long long tail_tiles, int splits) {
  if (!a->workspace || !aligned16(a->workspace)) return false;
  return tail_tiles * NUM_EPI_WARPS * 4 <= TAIL_CNT_BYTES &&
         TAIL_CNT_BYTES + tail_tiles * splits * (long long)BM * BN * 4 <= a->workspace_bytes;
}
// The tiles of a partly filled last wave are cut along K (see map_unit).  Model, in k-block times of one tile: a unit costs
// its k-blocks + c0 (fill / drain / epilogue); a tail unit additionally the fp32 round trip through L2 (c_fix).
static void plan_tail(GemmParams& p, const dvla_gemm_args* a, long long total_tiles, int slots) {
  if (!p.staged_ok || p.k_splits != 1 || total_tiles <= 0) return;
  const long long full_waves = total_tiles / slots;
  const long long rem = total_tiles - full_waves * slots;
  // Only GEMMs of at least one full wave: a row's result then depends on M only for the large training GEMMs.  Below one
  // wave (every GEMM of action inference) each output row is computed in the same K order whatever the batch it is in --
  // the incremental rollout's "bit-identical to the full window" property (tests/test_rollout_gpu.py) rests on that.
  if (rem == 0 || full_waves == 0) return;
  int tsp = (int)(slots / rem);
  if (tsp > 8) tsp = 8;
  if (tsp > p.num_k_blocks / 4) tsp = p.num_k_blocks / 4;
  if (tsp < 2) return;
  const int kbps = (p.num_k_blocks + tsp - 1) / tsp;
  tsp = (p.num_k_blocks + kbps - 1) / kbps;
  if (tsp < 2) return;
  // fixed cost per unit and of the fp32 fix-up, in k-block times of one tile (model constants, not re-tuned on the H100)
  const float c0 = 8.f, c_fix = 20.f;
  const float now = (float)(full_waves + 1) * ((float)p.num_k_blocks + c0);
  const float with_tail = (float)full_waves * ((float)p.num_k_blocks + c0) + (float)kbps + c0 + c_fix;
  if (with_tail > 0.93f * now) return;
  if (!tail_fits(a, rem, tsp)) return;
  p.tail_first = (int)(full_waves * slots); p.tail_splits = tsp; p.tail_kbps = kbps;
  p.tail_cnt = reinterpret_cast<unsigned*>(a->workspace);
  p.tail_ws = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(a->workspace) + TAIL_CNT_BYTES);
}

}  // namespace dvla

using namespace dvla;

extern "C" int dvla_gemm(const dvla_gemm_args* a, void* stream) {
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!a || !a->a || !a->b || !a->out) { set_error("dvla_gemm: null pointer"); return DVLA_ERR_INVALID; }
  if (a->M <= 0 || a->N <= 0 || a->K <= 0) { set_error("dvla_gemm: non-positive dims M=%lld N=%lld K=%lld", (long long)a->M, (long long)a->N, (long long)a->K); return DVLA_ERR_INVALID; }
  if (a->aux_in && a->aux_out) { set_error("dvla_gemm: aux_in and aux_out are exclusive"); return DVLA_ERR_INVALID; }
  if (!dropout_rate_ok(a->dropout_p)) { set_error("dvla_gemm: dropout_p out of range"); return DVLA_ERR_INVALID; }
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.out = a->out; p.bias = (const bf16*)a->bias; p.residual = a->residual;
  p.aux_out = (bf16*)a->aux_out; p.aux_in = (const bf16*)a->aux_in;
  p.M = (int)a->M; p.N = (int)a->N; p.K = (int)a->K;
  p.ldo = a->ldo; p.ldr = a->ldr; p.ld_aux = a->ld_aux;
  p.act = a->act; p.out_fp32 = a->out_fp32; p.alpha = a->alpha;
  if (a->dropout_p > 0.f) {
    dropout_thresh_scale(a->dropout_p, &p.drop_thresh, &p.drop_scale);
    p.drop_seed = a->dropout_seed;
    p.drop_seed_ptr = a->dropout_seed_ptr;
  }
  const int oal = a->out_fp32 ? 4 : 8;
  p.vec_ok = aligned16(a->out) && (a->ldo % oal == 0) &&
             (!a->bias || aligned16(a->bias)) &&
             (!a->residual || (aligned16(a->residual) && a->ldr % oal == 0)) &&
             (!a->aux_out || (aligned16(a->aux_out) && a->ld_aux % 8 == 0)) &&
             (!a->aux_in || (aligned16(a->aux_in) && a->ld_aux % 8 == 0));
  p.staged_ok = p.vec_ok && !a->out_fp32 && (a->N % 8 == 0);
  p.num_m_tiles = (p.M + BM - 1) / BM;
  p.num_n_tiles = (p.N + BN - 1) / BN;
  p.num_k_blocks = (p.K + BK - 1) / BK;

  const bool tma_ok = aligned16(a->a) && aligned16(a->b) && (a->lda % 8 == 0) && (a->ldb % 8 == 0);
  if (!tma_ok) {
    const long long groups = (long long)p.M * ((p.N + 7) / 8);
    const int threads = 128;
    if (g_plan) {
      const bool warp_kernel = p.K >= 128 && groups <= 65536;
      record_plan(p, warp_kernel ? 1 : 0, 1, 8, p.M, (int)(((warp_kernel ? groups * 32 : groups) + threads - 1) / threads));
      return DVLA_OK;
    }
    if (p.K >= 128 && groups <= 65536) {      // long contraction, small output: one warp per output group
      const long long blocks = (groups * 32 + threads - 1) / threads;
      gemm_simt_warp_kernel<<<(unsigned)blocks, threads, 0, s>>>((const bf16*)a->a, (const bf16*)a->b, a->lda, a->ldb,
                                                               a->a_mn_major, a->b_mn_major, p);
    } else {
      const long long blocks = (groups + threads - 1) / threads;
      gemm_simt_kernel<<<(unsigned)blocks, threads, 0, s>>>((const bf16*)a->a, (const bf16*)a->b, a->lda, a->ldb,
                                                          a->a_mn_major, a->b_mn_major, p);
    }
    DVLA_CHECK_LAUNCH("gemm_simt");
    return DVLA_OK;
  }
  const int sms = num_sms();
  const long long tiles = (long long)p.num_m_tiles * p.num_n_tiles;
  p.k_splits = 1;
  p.kb_per_split = p.num_k_blocks;
  // Split-K for pure accumulations (out += A.B: the weight-gradient GEMMs, few output tiles and a very long contraction):
  // work unit = (tile, k-range), partial sums added with red.global.add.bf16x2.  Pick the split with the lowest modelled
  // time = waves x (k-blocks per unit + fixed per-unit cost).
  const bool accum_only = p.staged_ok && a->residual == a->out && a->ldr == a->ldo && !a->bias && !a->aux_in &&
                          !a->aux_out && a->act == DVLA_ACT_NONE && a->dropout_p == 0.f;
  if (accum_only && splitk_enabled() && p.num_k_blocks >= 32) {
    const int smax = p.num_k_blocks / 16 < 16 ? p.num_k_blocks / 16 : 16;
    const float c0 = 8.f;
    float best = 1e30f; int best_s = 1;
    for (int sp = 1; sp <= smax; ++sp) {
      const int kbps = (p.num_k_blocks + sp - 1) / sp;
      const int se = (p.num_k_blocks + kbps - 1) / kbps;
      if (se != sp) continue;
      const long long waves = (tiles * sp + sms - 1) / sms;
      const float t = (float)waves * ((float)kbps + c0);
      if (t < best * 0.97f) { best = t; best_s = sp; }
    }
    if (best_s > 1) {
      p.k_splits = best_s;
      p.kb_per_split = (p.num_k_blocks + best_s - 1) / best_s;
      p.atomic_out = 1;
      p.residual = nullptr;
      return launch_tc_any(a, p, s);
    }
  }
  plan_tail(p, a, tiles, sms);
  return launch_tc_any(a, p, s);
}

extern "C" int dvla_gemm_plan(const dvla_gemm_args* a, dvla_gemm_plan_info* out) {
  if (!out) { set_error("dvla_gemm_plan: null output"); return DVLA_ERR_INVALID; }
  memset(out, 0, sizeof(*out));
  g_plan = out;
  const int rc = dvla_gemm(a, nullptr);
  g_plan = nullptr;
  return rc;
}
extern "C" int dvla_gemm_plan_unit(const dvla_gemm_plan_info* plan, int32_t unit, int32_t* tile, int32_t* kb0, int32_t* kb1,
                                   int32_t* slot, int32_t* split) {
  if (!plan || plan->kernel < 2 || unit < 0 || unit >= plan->units) { set_error("dvla_gemm_plan_unit: bad plan / unit"); return DVLA_ERR_INVALID; }
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.num_k_blocks = plan->k_blocks; p.k_splits = plan->k_splits; p.kb_per_split = plan->kb_per_split;
  p.tail_first = plan->tail_first; p.tail_splits = plan->tail_splits; p.tail_kbps = plan->tail_kbps;
  const Unit u = map_unit(unit, plan->m_tiles * plan->n_tiles, p);
  if (tile) *tile = u.tile;
  if (kb0) *kb0 = u.kb0;
  if (kb1) *kb1 = u.kb1;
  if (slot) *slot = u.slot;
  if (split) *split = u.split;
  return DVLA_OK;
}

extern "C" int64_t dvla_gemm_workspace_bytes(const dvla_gemm_args*) { return TAIL_CNT_BYTES + TAIL_WS_SLICES * BM * BN * 4; }
