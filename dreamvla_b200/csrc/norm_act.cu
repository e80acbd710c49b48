// HBM-bound row kernels: LayerNorm fwd/bwd, column sums (bias grads), dropout, activation backward, fp32->bf16 folds.
// One warp per row, 16-byte vector accesses, grids sized against the SM count.
#include "common.cuh"
#include "host.cuh"
#include "../../include/dvla.h"

namespace dvla {

// ------------------------------------------------------------------------------------------------------------------
// LayerNorm forward: warp per row; row cached in registers (D <= 1024) => one HBM read + one write per element.
// ------------------------------------------------------------------------------------------------------------------
template <int NV>  // NV = ceil(D / 256): 16-byte vectors per lane
__global__ void __launch_bounds__(256) layernorm_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ gamma,
                                                            const bf16* __restrict__ beta, bf16* __restrict__ y,
                                                            float* __restrict__ mean_out, float* __restrict__ rstd_out,
                                                            long long rows, int D, long long ldx, long long ldy, float eps) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nvec = D >> 3;
  for (long long row = static_cast<long long>(blockIdx.x) * 8 + warp; row < rows; row += static_cast<long long>(gridDim.x) * 8) {
    const bf16* xr = x + row * ldx;
    float v[NV][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        load_bf16x8(xr + vi * 8, v[i]);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += v[i][j];
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[i][j] = 0.f;
      }
    }
    const float mean = warp_sum(s) / D;
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { const float d = v[i][j] - mean; ss += d * d; }
      }
    }
    const float rstd = rsqrtf(warp_sum(ss) / D + eps);
    if (lane == 0) {
      if (mean_out) mean_out[row] = mean;
      if (rstd_out) rstd_out[row] = rstd;
    }
    bf16* yr = y + row * ldy;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        float o[8];
        float gm[8], bt[8];
        if (gamma) load_bf16x8(gamma + vi * 8, gm);
        if (beta) load_bf16x8(beta + vi * 8, bt);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float t = (v[i][j] - mean) * rstd;
          if (gamma) t *= gm[j];
          if (beta) t += bt[j];
          o[j] = t;
        }
        store_bf16x8(yr + vi * 8, o);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// LayerNorm backward: warp per row for dx; per-lane register partials for dgamma/dbeta, folded through shared memory
// and one fp32 atomicAdd per column per CTA.
// ------------------------------------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(256, 2) layernorm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                                                            const bf16* __restrict__ gamma, const float* __restrict__ mean,
                                                            const float* __restrict__ rstd, bf16* __restrict__ dx,
                                                            float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                            long long rows, int D, long long ld,
                                                            const bf16* __restrict__ dres) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nvec = D >> 3;
  float pg[NV][8], pb[NV][8];
#pragma unroll
  for (int i = 0; i < NV; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) { pg[i][j] = 0.f; pb[i][j] = 0.f; }

  // The row is kept as the RAW bf16 vectors it was loaded as (8 registers per 16 B of x and dy instead of 16 fp32) and
  // unpacked twice: with the dgamma/dbeta partials that fits 128 registers, i.e. two CTAs per SM and twice the loads in
  // flight of this latency-bound, HBM-limited kernel.
  for (long long row = static_cast<long long>(blockIdx.x) * 8 + warp; row < rows; row += static_cast<long long>(gridDim.x) * 8) {
    uint4 xr[NV], dr[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        xr[i] = __ldg(reinterpret_cast<const uint4*>(x + row * ld + vi * 8));
        dr[i] = __ldg(reinterpret_cast<const uint4*>(dy + row * ld + vi * 8));
      } else {
        xr[i] = make_uint4(0, 0, 0, 0);
        dr[i] = make_uint4(0, 0, 0, 0);
      }
    }
    const float mu = mean[row], rs = rstd[row];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        float xv[8], dv[8], gm[8];
        unpack_bf16x8(xr[i], xv);
        unpack_bf16x8(dr[i], dv);
        if (gamma) load_bf16x8(gamma + vi * 8, gm);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float h = (xv[j] - mu) * rs;
          pg[i][j] += dv[j] * h;
          pb[i][j] += dv[j];
          const float gd = gamma ? dv[j] * gm[j] : dv[j];
          s1 += gd;
          s2 += gd * h;
        }
      }
    }
    s1 = warp_sum(s1) / D;
    s2 = warp_sum(s2) / D;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        float xv[8], dv[8], gm[8], o[8];
        unpack_bf16x8(xr[i], xv);
        unpack_bf16x8(dr[i], dv);
        if (gamma) load_bf16x8(gamma + vi * 8, gm);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float h = (xv[j] - mu) * rs;
          const float gd = gamma ? dv[j] * gm[j] : dv[j];
          o[j] = rs * (gd - s1 - h * s2);
        }
        if (dres) {                                   // + gradient of the residual branch that forked at x
          float r8[8];
          load_bf16x8(dres + row * ld + vi * 8, r8);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += r8[j];
        }
        store_bf16x8(dx + row * ld + vi * 8, o);
      }
    }
  }
  if (dgamma || dbeta) {
    __shared__ float red[8][32 * 8 + 1];
    for (int pass = 0; pass < 2; ++pass) {
      float* dst = pass == 0 ? dgamma : dbeta;
      if (!dst) continue;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 8; ++j) red[warp][lane * 8 + j] = pass == 0 ? pg[i][j] : pb[i][j];
        __syncthreads();
        // 256 threads fold 8 warps for the 256 columns of this vector slab
        const int colv = threadIdx.x;  // 0..255 -> lane*8+j
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) t += red[w][colv];
        const int col = (colv >> 3) * 8 + i * 256 + (colv & 7);
        if (col < D) atomicAdd(dst + col, t);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// LayerNorm backward, version 2 (D a multiple of 256, with dgamma/dbeta): the kernel above is latency-bound on the decoders'
// [42400, 1024] tensors because a row costs two dependent
// round trips (x, dy -> reduce -> dres) and its 64 per-lane dgamma/dbeta partials cap residency at 16 warps per SM.  Here the
// partials live in SHARED memory (one private [2][D] fp32 slab per warp, plain read-modify-write with 16-byte accesses), the
// residual-branch gradient is fetched with x and dy (one round trip per row); 2 CTAs per SM without spills (3 would need <= 85 registers).
// ------------------------------------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(256, 2) layernorm_bwd_v2_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                                                                  const bf16* __restrict__ gamma, const float* __restrict__ mean,
                                                                  const float* __restrict__ rstd, bf16* __restrict__ dx,
                                                                  float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                                  long long rows, long long ld, const bf16* __restrict__ dres) {
  constexpr int D = NV * 256;
  extern __shared__ __align__(16) float ln_acc[];                  // [8 warps][2][D]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* ag = ln_acc + warp * 2 * D;
  float* ab = ag + D;
  for (int i = lane; i < 2 * D; i += 32) ag[i] = 0.f;
  __syncwarp();
  auto load_gamma = [&](int i, float (&g)[8]) {       // 2 KB, L1 resident: cheaper than 8 * NV registers per lane
    if (gamma) load_bf16x8(gamma + (lane + i * 32) * 8, g);
    else {
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] = 1.f;
    }
  };
  for (long long row = static_cast<long long>(blockIdx.x) * 8 + warp; row < rows; row += static_cast<long long>(gridDim.x) * 8) {
    uint4 xr[NV], dr[NV], rr[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const long long off = row * ld + (lane + i * 32) * 8;
      xr[i] = __ldg(reinterpret_cast<const uint4*>(x + off));
      dr[i] = __ldg(reinterpret_cast<const uint4*>(dy + off));
      rr[i] = dres ? __ldg(reinterpret_cast<const uint4*>(dres + off)) : make_uint4(0, 0, 0, 0);
    }
    const float mu = mean[row], rs = rstd[row];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      float xv[8], dv[8], gmv[8];
      unpack_bf16x8(xr[i], xv);
      unpack_bf16x8(dr[i], dv);
      load_gamma(i, gmv);
      const int c0 = (lane + i * 32) * 8;
      float4 g0 = *reinterpret_cast<float4*>(ag + c0), g1 = *reinterpret_cast<float4*>(ag + c0 + 4);
      float4 b0 = *reinterpret_cast<float4*>(ab + c0), b1 = *reinterpret_cast<float4*>(ab + c0 + 4);
      float hh[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        hh[j] = (xv[j] - mu) * rs;
        const float gd = dv[j] * gmv[j];
        s1 += gd;
        s2 = fmaf(gd, hh[j], s2);
      }
      g0.x = fmaf(dv[0], hh[0], g0.x); g0.y = fmaf(dv[1], hh[1], g0.y); g0.z = fmaf(dv[2], hh[2], g0.z); g0.w = fmaf(dv[3], hh[3], g0.w);
      g1.x = fmaf(dv[4], hh[4], g1.x); g1.y = fmaf(dv[5], hh[5], g1.y); g1.z = fmaf(dv[6], hh[6], g1.z); g1.w = fmaf(dv[7], hh[7], g1.w);
      b0.x += dv[0]; b0.y += dv[1]; b0.z += dv[2]; b0.w += dv[3];
      b1.x += dv[4]; b1.y += dv[5]; b1.z += dv[6]; b1.w += dv[7];
      *reinterpret_cast<float4*>(ag + c0) = g0; *reinterpret_cast<float4*>(ag + c0 + 4) = g1;
      *reinterpret_cast<float4*>(ab + c0) = b0; *reinterpret_cast<float4*>(ab + c0 + 4) = b1;
    }
    s1 = warp_sum(s1) * (1.0f / D);
    s2 = warp_sum(s2) * (1.0f / D);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      float xv[8], dv[8], r8[8], o[8], gmv[8];
      unpack_bf16x8(xr[i], xv);
      unpack_bf16x8(dr[i], dv);
      unpack_bf16x8(rr[i], r8);
      load_gamma(i, gmv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float h = (xv[j] - mu) * rs;
        o[j] = fmaf(rs, dv[j] * gmv[j] - s1 - h * s2, r8[j]);
      }
      store_bf16x8(dx + row * ld + (lane + i * 32) * 8, o);
    }
  }
  __syncthreads();
  // fold the 8 per-warp slabs; one fp32 atomic per column per CTA
  for (int c = threadIdx.x; c < 2 * D; c += 256) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += ln_acc[w * 2 * D + c];
    float* dst = c < D ? dgamma : dbeta;
    if (dst) atomicAdd(dst + (c < D ? c : c - D), t);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Column sum (bias gradient): out[n] += sum_r x[r, n]
// Block = 8 warps over a slab of 256 columns x a chunk of rows: each lane keeps 8 column partials in registers (coalesced
// 512 B per warp per row), the 8 warps fold through shared memory, ONE fp32 atomicAdd per column per block.
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) colsum_kernel(const bf16* __restrict__ x, long long rows, int N, long long ld,
                                                     float* __restrict__ out, int rows_per_block, int vec) {
  const long long r0 = static_cast<long long>(blockIdx.y) * rows_per_block;
  const long long r1 = min(rows, r0 + rows_per_block);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __shared__ float red[8][257];
  if (vec) {
    const int col = blockIdx.x * 256 + lane * 8;
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (col < N) {
      long long r = r0 + warp;
      for (; r + 24 < r1; r += 32) {            // 4 independent 16-byte loads in flight per lane
        uint4 u[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) u[k] = __ldg(reinterpret_cast<const uint4*>(x + (r + 8 * k) * ld + col));
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float2 t;
          t = unpack_bf16x2(u[k].x); acc[0] += t.x; acc[1] += t.y;
          t = unpack_bf16x2(u[k].y); acc[2] += t.x; acc[3] += t.y;
          t = unpack_bf16x2(u[k].z); acc[4] += t.x; acc[5] += t.y;
          t = unpack_bf16x2(u[k].w); acc[6] += t.x; acc[7] += t.y;
        }
      }
      for (; r < r1; r += 8) {
        float f[8];
        load_bf16x8(x + r * ld + col, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += f[j];
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) red[warp][lane * 8 + j] = acc[j];
  } else {
    const int col = blockIdx.x * 256 + threadIdx.x;   // scalar path: thread per column, all rows of the chunk
    float acc = 0.f;
    if (col < N)
      for (long long r = r0; r < r1; ++r) acc += __bfloat162float(x[r * ld + col]);
    if (col < N) atomicAdd(out + col, acc);
    return;
  }
  __syncthreads();
  const int c = threadIdx.x;
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) t += red[w][c];
  const int col = blockIdx.x * 256 + c;
  if (col < N) atomicAdd(out + col, t);
}

// ------------------------------------------------------------------------------------------------------------------
__global__ void accum_fp32_into_bf16_kernel(const float* __restrict__ src, bf16* __restrict__ dst, long long n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    dst[i] = __float2bfloat16(__bfloat162float(dst[i]) + src[i]);
}

// ------------------------------------------------------------------------------------------------------------------
// Dropout with the GEMM-epilogue mask convention: RNG block = row*ceil(N/8) + col/8, bit col%8.
// ------------------------------------------------------------------------------------------------------------------
__global__ void dropout_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, long long rows, int N, long long ldx,
                               long long ldy, uint32_t thresh, float scale, uint64_t seed0,
                               const uint64_t* __restrict__ seed_ptr, int vec) {
  const uint64_t seed = seed0 + (seed_ptr ? __ldg(seed_ptr) : 0ull);
  const int groups = (N + 7) >> 3;
  const long long total = rows * groups;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / groups;
    const int col = static_cast<int>(i % groups) * 8;
    const uint32_t keep = dropout_keep8(seed, static_cast<uint64_t>(i), thresh);
    if (vec) {
      float f[8];
      load_bf16x8(x + row * ldx + col, f);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = ((keep >> j) & 1u) ? f[j] * scale : 0.f;
      store_bf16x8(y + row * ldy + col, f);
    } else {
      for (int j = 0; j < 8 && col + j < N; ++j) {
        const float f = __bfloat162float(x[row * ldx + col + j]);
        y[row * ldy + col + j] = __float2bfloat16(((keep >> j) & 1u) ? f * scale : 0.f);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// dx = dy * act'(pre): HBM-bound (2 reads + 1 write of 2 B per element); 8 elements (16 B) per thread per access, the
// activation switch hoisted out of the element loop (act_bwd_mul_n)
__global__ void __launch_bounds__(256) act_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ pre,
                                                      bf16* __restrict__ dx, long long n, int act) {
  const long long nvec = n >> 3;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const uint4* dy4 = reinterpret_cast<const uint4*>(dy);
  const uint4* pre4 = reinterpret_cast<const uint4*>(pre);
  uint4* dx4 = reinterpret_cast<uint4*>(dx);
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    float v[8], x[8];
    unpack_bf16x8(__ldg(dy4 + i), v);
    unpack_bf16x8(__ldg(pre4 + i), x);
    act_bwd_mul_n<8>(v, x, act);
    dx4[i] = pack_bf16x8(v);
  }
  for (long long i = (nvec << 3) + static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
    dx[i] = __float2bfloat16(__bfloat162float(dy[i]) * act_bwd(__bfloat162float(pre[i]), act));
}
__global__ void act_bwd_scalar_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ pre, bf16* __restrict__ dx,
                                      long long n, int act) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    dx[i] = __float2bfloat16(__bfloat162float(dy[i]) * act_bwd(__bfloat162float(pre[i]), act));
}

// ------------------------------------------------------------------------------------------------------------------
// dx = dy * act'(pre) AND colsum[c] += sum_r dx[r, c] in one pass: the bias gradient of the first MLP layer is the column
// sum of exactly the tensor this kernel writes, so the separate colsum pass (a third read of [rows, 4D]) disappears.
// Same block shape as colsum_kernel: 8 warps over a slab of 256 columns x a chunk of rows, each lane owns 8 columns
// (one 16-byte vector of dy and of pre per row, 4 rows in flight), column partials in registers -> shared memory -> ONE
// fp32 atomicAdd per column per block.  The sum is taken over the fp32 products (before the bf16 rounding of dx).
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) act_bwd_colsum_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ pre,
                                                             bf16* __restrict__ dx, long long rows, int N,
                                                             float* __restrict__ colsum, int rows_per_block, int act) {
  const long long r0 = static_cast<long long>(blockIdx.y) * rows_per_block;
  const long long r1 = min(rows, r0 + rows_per_block);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __shared__ float red[8][257];
  const int col = blockIdx.x * 256 + lane * 8;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  auto one = [&](const uint4& a, const uint4& b, long long r) {
    float v[8], x[8];
    unpack_bf16x8(a, v);
    unpack_bf16x8(b, x);
    act_bwd_mul_n<8>(v, x, act);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += v[j];
    store_bf16x8(dx + r * N + col, v);
  };
  if (col < N) {
    long long r = r0 + warp;
    for (; r + 24 < r1; r += 32) {
      uint4 a[4], b[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        a[k] = __ldg(reinterpret_cast<const uint4*>(dy + (r + 8 * k) * N + col));
        b[k] = __ldg(reinterpret_cast<const uint4*>(pre + (r + 8 * k) * N + col));
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) one(a[k], b[k], r + 8 * k);
    }
    for (; r < r1; r += 8)
      one(__ldg(reinterpret_cast<const uint4*>(dy + r * N + col)), __ldg(reinterpret_cast<const uint4*>(pre + r * N + col)), r);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[warp][lane * 8 + j] = acc[j];
  __syncthreads();
  const int c = threadIdx.x;
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) t += red[w][c];
  if (blockIdx.x * 256 + c < N) atomicAdd(colsum + blockIdx.x * 256 + c, t);
}

// ------------------------------------------------------------------------------------------------------------------
// out[s, :a] = e[s], out[s, a:] = m: per-sequence rows followed by rows shared by every sequence (16-byte vectors)
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) cat_broadcast_kernel(const uint4* __restrict__ e, const uint4* __restrict__ m,
                                                            uint4* __restrict__ out, long long n, int a, int b, int c8) {
  const long long per_seq = static_cast<long long>(a + b) * c8;
  const long long total = n * per_seq;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long s = i / per_seq;
    const long long r = i - s * per_seq;
    const long long ea = static_cast<long long>(a) * c8;
    out[i] = r < ea ? e[s * ea + r] : __ldg(m + (r - ea));
  }
}

// Calls f(std::integral_constant<int, NV>()) for the LayerNorm kernels' NV = ceil(D / 256) in 1..4 (D <= 1024).
template <class F>
static auto with_nv(int nv, F f) {
  switch (nv) {
    case 1: return f(std::integral_constant<int, 1>());
    case 2: return f(std::integral_constant<int, 2>());
    case 3: return f(std::integral_constant<int, 3>());
    default: return f(std::integral_constant<int, 4>());
  }
}

}  // namespace dvla

using namespace dvla;

extern "C" int dvla_layernorm_fwd(const dvla_layernorm_fwd_args* a, void* stream) {
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!a || !a->x || !a->y) { set_error("layernorm_fwd: null pointer"); return DVLA_ERR_INVALID; }
  if (a->D % 8 || a->ldx % 8 || a->ldy % 8 || a->D > 1024 || a->D <= 0) {
    set_error("layernorm_fwd: need D%%8==0, D<=1024, strides%%8==0 (D=%lld)", (long long)a->D);
    return DVLA_ERR_UNSUPPORTED;
  }
  if (a->rows <= 0) return DVLA_OK;
  const unsigned blocks = grid_for(a->rows, 8, 8);
  with_nv((int)((a->D + 255) / 256), [&](auto NV) {
    layernorm_fwd_kernel<NV><<<blocks, 256, 0, s>>>((const bf16*)a->x, (const bf16*)a->gamma, (const bf16*)a->beta, (bf16*)a->y,
                                                     a->mean, a->rstd, a->rows, (int)a->D, a->ldx, a->ldy, a->eps);
  });
  DVLA_CHECK_LAUNCH("layernorm_fwd");
  return DVLA_OK;
}

extern "C" int dvla_layernorm_bwd(const dvla_layernorm_bwd_args* a, void* stream) {
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!a || !a->dy || !a->x || !a->mean || !a->rstd || !a->dx) { set_error("layernorm_bwd: null pointer"); return DVLA_ERR_INVALID; }
  if (a->D % 8 || a->ld % 8 || a->D > 1024 || a->D <= 0) {
    set_error("layernorm_bwd: need D%%8==0, D<=1024, ld%%8==0 (D=%lld)", (long long)a->D);
    return DVLA_ERR_UNSUPPORTED;
  }
  if (a->rows <= 0) return DVLA_OK;
  const int nv = (int)((a->D + 255) / 256);
  const unsigned blocks = grid_for(a->rows, 8, 2);   // 2 resident blocks per SM; 2*D fp32 atomics per block at the end
  if (a->D % 256 == 0 && (a->dgamma || a->dbeta) && a->rows >= 2048) {
    const int rc = with_nv(nv, [&](auto NV) {
      constexpr int smem = 8 * 2 * NV * 256 * sizeof(float);
      static std::once_flag once;
      static cudaError_t attr_err;
      if (!set_smem_attr_once(once, attr_err, layernorm_bwd_v2_kernel<NV>, smem)) {
        set_error("layernorm_bwd_v2 smem attr: %s", cudaGetErrorString(attr_err));
        return DVLA_ERR_CUDA;
      }
      layernorm_bwd_v2_kernel<NV><<<blocks, 256, smem, s>>>((const bf16*)a->dy, (const bf16*)a->x, (const bf16*)a->gamma, a->mean,
                                                            a->rstd, (bf16*)a->dx, a->dgamma, a->dbeta, a->rows, a->ld,
                                                            (const bf16*)a->dres);
      return DVLA_OK;
    });
    if (rc != DVLA_OK) return rc;
    DVLA_CHECK_LAUNCH("layernorm_bwd_v2");
    return DVLA_OK;
  }
  with_nv(nv, [&](auto NV) {
    layernorm_bwd_kernel<NV><<<blocks, 256, 0, s>>>((const bf16*)a->dy, (const bf16*)a->x, (const bf16*)a->gamma, a->mean, a->rstd,
                                                     (bf16*)a->dx, a->dgamma, a->dbeta, a->rows, (int)a->D, a->ld,
                                                     (const bf16*)a->dres);
  });
  DVLA_CHECK_LAUNCH("layernorm_bwd");
  return DVLA_OK;
}

extern "C" int dvla_colsum_accum(const void* x, int64_t rows, int64_t N, int64_t ld, float* out, void* stream) {
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!x || !out) { set_error("colsum: null pointer"); return DVLA_ERR_INVALID; }
  if (rows <= 0 || N <= 0) return DVLA_OK;
  const int vec = (N % 8 == 0) && (ld % 8 == 0) && aligned16(x);
  int rpb;
  const dim3 grid = slab_grid(rows, N, 6, 64, &rpb);    // ~6 blocks of 256 threads per SM: enough loads in flight for HBM
  colsum_kernel<<<grid, 256, 0, s>>>((const bf16*)x, rows, (int)N, ld, out, rpb, vec);
  DVLA_CHECK_LAUNCH("colsum");
  return DVLA_OK;
}

extern "C" int dvla_accum_fp32_into_bf16(const float* src, void* dst, int64_t n, void* stream) {
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!src || !dst) { set_error("accum_fp32_into_bf16: null pointer"); return DVLA_ERR_INVALID; }
  if (n <= 0) return DVLA_OK;
  accum_fp32_into_bf16_kernel<<<grid_for(n, 256, 4), 256, 0, s>>>(src, (bf16*)dst, n);
  DVLA_CHECK_LAUNCH("accum_fp32_into_bf16");
  return DVLA_OK;
}

extern "C" int dvla_dropout(const void* x, void* y, int64_t rows, int64_t N, int64_t ldx, int64_t ldy, float p, uint64_t seed,
                            const uint64_t* seed_ptr, void* stream) {
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!x || !y) { set_error("dropout: null pointer"); return DVLA_ERR_INVALID; }
  if (!dropout_rate_ok(p)) { set_error("dropout: p out of range"); return DVLA_ERR_INVALID; }
  if (rows <= 0 || N <= 0) return DVLA_OK;
  uint32_t thresh;
  float scale;
  dropout_thresh_scale(p, &thresh, &scale);
  const int vec = (N % 8 == 0) && (ldx % 8 == 0) && (ldy % 8 == 0) && aligned16(x, y);
  dropout_kernel<<<grid_for(rows * ((N + 7) / 8), 256, 8), 256, 0, s>>>((const bf16*)x, (bf16*)y, rows, (int)N, ldx, ldy, thresh, scale, seed, seed_ptr, vec);
  DVLA_CHECK_LAUNCH("dropout");
  return DVLA_OK;
}

extern "C" int dvla_act_bwd(const void* dy, const void* pre, void* dx, int64_t n, int32_t act, void* stream) {
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!dy || !pre || !dx) { set_error("act_bwd: null pointer"); return DVLA_ERR_INVALID; }
  if (n <= 0) return DVLA_OK;
  const bool vec = aligned16(dy, pre, dx);
  const unsigned blocks = grid_for(vec ? (n + 7) / 8 : n, 256, 8);
  if (vec) act_bwd_kernel<<<blocks, 256, 0, s>>>((const bf16*)dy, (const bf16*)pre, (bf16*)dx, n, act);
  else     act_bwd_scalar_kernel<<<blocks, 256, 0, s>>>((const bf16*)dy, (const bf16*)pre, (bf16*)dx, n, act);
  DVLA_CHECK_LAUNCH("act_bwd");
  return DVLA_OK;
}

extern "C" int dvla_act_bwd_colsum(const void* dy, const void* pre, void* dx, int64_t rows, int64_t N, int32_t act, float* colsum,
                                   void* stream) {
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!dy || !pre || !dx || !colsum) { set_error("act_bwd_colsum: null pointer"); return DVLA_ERR_INVALID; }
  if (rows <= 0 || N <= 0) return DVLA_OK;
  if (N % 8 || !aligned16(dy, pre, dx)) {
    // unaligned / odd width: the two separate passes
    int rc = dvla_act_bwd(dy, pre, dx, rows * N, act, stream);
    if (rc != DVLA_OK) return rc;
    return dvla_colsum_accum(dx, rows, N, N, colsum, stream);
  }
  int rpb;
  const dim3 grid = slab_grid(rows, N, 8, 32, &rpb);
  act_bwd_colsum_kernel<<<grid, 256, 0, s>>>((const bf16*)dy, (const bf16*)pre, (bf16*)dx, rows, (int)N, colsum, rpb, act);
  DVLA_CHECK_LAUNCH("act_bwd_colsum");
  return DVLA_OK;
}

extern "C" int dvla_cat_broadcast(const void* e, const void* m, void* out, int64_t n, int64_t a, int64_t b, int64_t C,
                                  void* stream) {
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!e || !m || !out) { set_error("cat_broadcast: null pointer"); return DVLA_ERR_INVALID; }
  if (n <= 0 || a < 0 || b <= 0 || C <= 0 || C % 8) { set_error("cat_broadcast: bad dims (C must be a multiple of 8)"); return DVLA_ERR_INVALID; }
  if (!aligned16(e, m, out)) { set_error("cat_broadcast: buffers must be 16-byte aligned"); return DVLA_ERR_INVALID; }
  cat_broadcast_kernel<<<grid_for(n * (a + b) * (C / 8), 256 * 4, 16), 256, 0, s>>>((const uint4*)e, (const uint4*)m, (uint4*)out, n, (int)a, (int)b, (int)(C / 8));
  DVLA_CHECK_LAUNCH("cat_broadcast");
  return DVLA_OK;
}
