// Whole-sampler kernel for action inference: the 10-step DDIM loop of the DiT action head with classifier-free guidance
// (reference models/dreamvla_model.py:935-987 -> action_model.py:76-83 -> gaussian_diffusion.py:522-569,609-689 ->
// models.py:234-268) as ONE persistent cooperative kernel.
//
// Why: at batch 1 the sampler is 10 x (12 DiT blocks + embedders + final layer + DDIM algebra) ~ 1100 kernel launches on
// 12 token rows (2 guidance branches x 6 tokens) -- every launch is latency, none is work: the whole DiT-B is 170 MB of bf16
// weights, i.e. ~30 us per pass at HBM speed.  The same kernel runs DiT-S (head_dim 96) and DiT-L (depth 24, hidden 1024).  Here one CTA per SM stays resident for the entire sample; every linear layer
// is a "skinny" GEMM (M <= 24 rows) in which a warp owns one output column, streams that column's weight row from HBM/L2
// with 16-byte loads and keeps the activations (bf16) in shared memory; the phases of a block (LN+QKV | attention+proj+res |
// LN+fc1+GELU | fc2+res) are separated by grid barriers (cooperative launch) instead of kernel boundaries.  Timestep and
// condition embeddings are hoisted out of the loop (they do not depend on x); x itself (T x 7 numbers per sample) lives in
// shared memory of every CTA and is advanced redundantly, so no barrier is needed for the final layer / guidance / DDIM update.
// Buffers exchanged between CTAs (h, qkv, u, te, ze) are read with ld.global.cg: L1 is not coherent across SMs.
//
// Numerics follow the module path where it rounds: GEMM inputs are bf16 (activations are rounded when staged in shared
// memory), accumulation fp32; the residual stream, LayerNorm statistics and softmax stay fp32 (the module path keeps the
// residual stream in bf16), so results agree with it to bf16 rounding, not bit for bit (tests/test_rollout_gpu.py).
#include <cooperative_groups.h>

#include <string.h>

#include "common.cuh"
#include "host.cuh"
#include "../../include/dvla.h"

namespace cg = cooperative_groups;

namespace dvla {
namespace {

constexpr int DS_THREADS = 512;      // 16 warps per SM: the skinny GEMMs hide weight-load latency with warps in flight
constexpr int DS_WARPS = DS_THREADS / 32;
constexpr int DS_MAXM = 12;          // rows: 2 guidance branches x bs x 2T tokens (bs = 1: the rollout case; larger batches use the module path)
constexpr int DS_MAX_DEPTH = 28;
constexpr int DS_MAX_STEPS = 16;

struct DitBlockW { const bf16 *qkv_w, *qkv_b, *proj_w, *proj_b, *fc1_w, *fc1_b, *fc2_w, *fc2_b; };
struct DitSamplerParams {
  DitBlockW blk[DS_MAX_DEPTH];
  int depth;
  const bf16 *x_w, *x_b, *t0_w, *t0_b, *t2_w, *t2_b, *z_w, *z_b, *uncond, *pos, *fin_w, *fin_b;
  const bf16* z;            // [bs, T, token]
  const float* noise;       // [bs, T, C]
  float* out;               // [bs, T, C]
  int tmap[DS_MAX_STEPS];
  float sqrt_recip[DS_MAX_STEPS], sqrt_recipm1[DS_MAX_STEPS], acp_prev[DS_MAX_STEPS];
  int n_steps;
  float cfg_scale;
  int bs, T, C, H, heads, token, mlp, freq;
  float *h0, *h1, *qkv, *u, *te, *t1, *ze;     // fp32 scratch (global, L2 resident)
};

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  float2 t;
  t = unpack_bf16x2(u.x); f[0] = t.x; f[1] = t.y;
  t = unpack_bf16x2(u.y); f[2] = t.x; f[3] = t.y;
  t = unpack_bf16x2(u.z); f[4] = t.x; f[5] = t.y;
  t = unpack_bf16x2(u.w); f[6] = t.x; f[7] = t.y;
}
__device__ __forceinline__ float gelu_tanh_f(float x) {
  const float u = 0.7978845608028654f * (x + 0.044715f * x * x * x);
  return 0.5f * x * (1.0f + tanhf(u));
}

// out(m, n) = sum_k Xs[m][k] * W[n][k] (+ bias[n]) for every column n owned by this warp; Xs: shared, bf16, [M][K], K % 8 == 0,
// M <= MROWS.  A warp works on TWO columns at a time (the staged activations are read once for both) and issues the weight
// loads of four 8-element chunks per column before using them: the kernel is a weight-streaming loop whose only latency
// hiding is loads in flight.  Lane m applies the epilogue of row m:
//   EPI_STORE out = v | EPI_SILU out = silu(v) | EPI_GELU out = gelu_tanh(v) | EPI_ACC out += v (ld.cg / st.cg: the residual
//   stream is exchanged between CTAs)
// ONE out-of-line copy per MROWS: inlined at its seven call sites the unrolled body did not fit the instruction cache
// (ncu of the first version: 27 % of warp cycles stalled on no_instruction, 4x the expected instruction count).
enum { EPI_STORE = 0, EPI_SILU = 1, EPI_GELU = 2, EPI_ACC = 3 };
template <int MROWS>
__device__ __noinline__ void skinny_gemm(const bf16* __restrict__ Xs, int M, int K, const bf16* __restrict__ W,
                                         const bf16* __restrict__ bias, int N, float* __restrict__ out, int ldo, int mode) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gw = blockIdx.x * DS_WARPS + warp, nw = gridDim.x * DS_WARPS;
  const int chunks = K >> 3;
  // Few output columns, long contraction (attention projection, fc2: N = hidden): several warps share a column, each takes a
  // K range and adds its partial sum with red.global.add.f32 (bias from range 0).  fp32 atomics: the order of the <= 4
  // partials is not fixed, so the sampler is reproducible to fp32 rounding, not bitwise.
  const int ksplit = (mode == EPI_ACC && nw >= 2 * N) ? (nw / N < 4 ? nw / N : 4) : 1;
  if (ksplit > 1) {
    for (int unit = gw; unit < N * ksplit; unit += nw) {
      const int n = unit % N, ks = unit / N;
      const int cb = (chunks * ks) / ksplit, ce = (chunks * (ks + 1)) / ksplit;
      float acc[MROWS];
#pragma unroll
      for (int m = 0; m < MROWS; ++m) acc[m] = 0.f;
      const uint4* wr = reinterpret_cast<const uint4*>(W + static_cast<long long>(n) * K);
      for (int c0 = cb + lane; c0 < ce; c0 += 128) {
        uint4 a[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) a[u] = (c0 + 32 * u) < ce ? __ldg(wr + c0 + 32 * u) : make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int c = c0 + 32 * u;
          if (c >= ce) continue;
          float wa[8];
          unpack8(a[u], wa);
#pragma unroll
          for (int m = 0; m < MROWS; ++m) {
            float x[8];
            unpack8(*reinterpret_cast<const uint4*>(Xs + (m < M ? m : 0) * K + c * 8), x);
            float s0 = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) s0 = fmaf(x[j], wa[j], s0);
            acc[m] += s0;
          }
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int m = 0; m < MROWS; ++m) acc[m] += __shfl_xor_sync(0xffffffffu, acc[m], o);
      float mine = 0.f;
#pragma unroll
      for (int m = 0; m < MROWS; ++m)
        if (lane == m) mine = acc[m];
      if (lane < M) atomicAdd(out + static_cast<long long>(lane) * ldo + n, mine + ((bias && ks == 0) ? __bfloat162float(bias[n]) : 0.f));
    }
    return;
  }
  for (int n0 = gw; n0 < N; n0 += 2 * nw) {
    const int n1 = n0 + nw;
    const bool two = n1 < N;
    float acc0[MROWS], acc1[MROWS];
#pragma unroll
    for (int m = 0; m < MROWS; ++m) { acc0[m] = 0.f; acc1[m] = 0.f; }
    const uint4* w0 = reinterpret_cast<const uint4*>(W + static_cast<long long>(n0) * K);
    const uint4* w1 = reinterpret_cast<const uint4*>(W + static_cast<long long>(two ? n1 : n0) * K);
    for (int c0 = lane; c0 < chunks; c0 += 128) {
      uint4 a[4], b[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int c = c0 + 32 * u;
        a[u] = c < chunks ? __ldg(w0 + c) : make_uint4(0, 0, 0, 0);
        b[u] = c < chunks ? __ldg(w1 + c) : make_uint4(0, 0, 0, 0);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int c = c0 + 32 * u;
        if (c >= chunks) continue;
        float wa[8], wb[8];
        unpack8(a[u], wa);
        unpack8(b[u], wb);
#pragma unroll
        for (int m = 0; m < MROWS; ++m) {
          float x[8];
          unpack8(*reinterpret_cast<const uint4*>(Xs + (m < M ? m : 0) * K + c * 8), x);
          float s0 = 0.f, s1 = 0.f;
#pragma unroll
          for (int j = 0; j < 8; ++j) { s0 = fmaf(x[j], wa[j], s0); s1 = fmaf(x[j], wb[j], s1); }
          acc0[m] += s0;
          acc1[m] += s1;
        }
      }
    }
    // butterfly over all rows in lock step (independent shuffles: throughput, not 2*MROWS dependent chains)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int m = 0; m < MROWS; ++m) {
        acc0[m] += __shfl_xor_sync(0xffffffffu, acc0[m], o);
        acc1[m] += __shfl_xor_sync(0xffffffffu, acc1[m], o);
      }
    }
    float mine0 = 0.f, mine1 = 0.f;
#pragma unroll
    for (int m = 0; m < MROWS; ++m)
      if (lane == m) { mine0 = acc0[m]; mine1 = acc1[m]; }
    if (lane < M) {
#pragma unroll 1
      for (int t = 0; t < (two ? 2 : 1); ++t) {
        const int n = t ? n1 : n0;
        float v = (t ? mine1 : mine0) + (bias ? __bfloat162float(bias[n]) : 0.f);
        float* dst = out + static_cast<long long>(lane) * ldo + n;
        if (mode == EPI_SILU) v = v / (1.0f + __expf(-v));
        else if (mode == EPI_GELU) v = gelu_tanh_f(v);
        else if (mode == EPI_ACC) v += __ldcg(dst);
        __stcg(dst, v);
      }
    }
  }
}

// Xs[m][:] = bf16(LayerNorm(h[m][:])) without affine, eps 1e-6 (timm Block with elementwise_affine=False).  Warp per row; the row
// is fetched ONCE with independent 16-byte ld.global.cg loads (up to 8 per lane, H <= 1024) and normalised from registers:
// three dependent scalar passes over L2 cost ~10 us per phase.
__device__ __forceinline__ void stage_layernorm_row(bf16* __restrict__ dst, const float* __restrict__ row, int H) {
  const int lane = threadIdx.x & 31;
  const int n4 = H >> 2;
  const float4* r4 = reinterpret_cast<const float4*>(row);
  float4 v[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const int i = lane + 32 * u;
    v[u] = i < n4 ? __ldcg(r4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float s = 0.f;
#pragma unroll
  for (int u = 0; u < 8; ++u) s += (v[u].x + v[u].y) + (v[u].z + v[u].w);
  const float mean = warp_sum_f(s) / H;
  float q = 0.f;
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    if (lane + 32 * u < n4) {
      const float a = v[u].x - mean, b = v[u].y - mean, c = v[u].z - mean, d = v[u].w - mean;
      q += (a * a + b * b) + (c * c + d * d);
    }
  }
  const float rstd = rsqrtf(warp_sum_f(q) / H + 1e-6f);
  uint2* d2 = reinterpret_cast<uint2*>(dst);
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const int i = lane + 32 * u;
    if (i < n4) d2[i] = make_uint2(pack_bf16x2((v[u].x - mean) * rstd, (v[u].y - mean) * rstd),
                                   pack_bf16x2((v[u].z - mean) * rstd, (v[u].w - mean) * rstd));
  }
}
__device__ __forceinline__ void stage_layernorm(bf16* Xs, const float* __restrict__ h, int M, int H) {
  const int warp = threadIdx.x >> 5;
  for (int m = warp; m < M; m += DS_WARPS) stage_layernorm_row(Xs + m * H, h + static_cast<long long>(m) * H, H);
}
__device__ __forceinline__ void stage_rows(bf16* Xs, const float* __restrict__ src, int n) {   // fp32 global -> bf16 shared, n % 4 == 0
  const float4* s4 = reinterpret_cast<const float4*>(src);
  uint2* d2 = reinterpret_cast<uint2*>(Xs);
  const int n4 = n >> 2;
  for (int i0 = threadIdx.x; i0 < n4; i0 += 6 * DS_THREADS) {
    float4 v[6];
#pragma unroll
    for (int u = 0; u < 6; ++u) {
      const int i = i0 + u * DS_THREADS;
      v[u] = i < n4 ? __ldcg(s4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 6; ++u) {
      const int i = i0 + u * DS_THREADS;
      if (i < n4) d2[i] = make_uint2(pack_bf16x2(v[u].x, v[u].y), pack_bf16x2(v[u].z, v[u].w));
    }
  }
}

// HD: head_dim (64: DiT-B / DiT-L, 96: DiT-S).  In the attention phase lane l holds dims 2l, 2l+1 of a head (float2) and,
// at HD = 96, also dim 64 + l.
template <int MROWS, int L, int HD>
__global__ void __launch_bounds__(DS_THREADS, 1) dit_ddim_sample_kernel(const __grid_constant__ DitSamplerParams p) {
  static_assert(HD == 64 || HD == 96, "head_dim 64 or 96");
  extern __shared__ __align__(16) uint8_t ds_smem[];
  cg::grid_group grid = cg::this_grid();
  const int H = p.H, T = p.T, C = p.C, bs = p.bs;
  // L = 2T tokens per sequence: T condition tokens + T action tokens (models.py:240-244)
  const int nseq = 2 * bs;             // guidance: sequences [0, bs) conditional, [bs, 2bs) unconditional (models.py:253-257)
  const int M = nseq * L;
  bf16* Xs = reinterpret_cast<bf16*>(ds_smem);                                // staged GEMM input, up to [M][mlp]
  float* xcur = reinterpret_cast<float*>(ds_smem + static_cast<size_t>(M) * p.mlp * 2);     // [bs][T][C] current sample
  float* eps_s = xcur + bs * T * C;                                           // [nseq][T][C] final-layer outputs
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int gtid = blockIdx.x * DS_THREADS + tid, gthreads = gridDim.x * DS_THREADS;

  // ---- prologue A: timestep-frequency features -> t1 = silu(W0 f + b0) for all steps;  ze = Wz z + bz for the bs*T condition
  //      rows and for the `uncondition` vector (row bs*T)
  for (int i = tid; i < p.n_steps * p.freq; i += DS_THREADS) {
    const int s = i / p.freq, k = i - s * p.freq, half = p.freq >> 1;
    const float fr = __expf(-9.210340371976184f * static_cast<float>(k < half ? k : k - half) / half);   // ln(10000)
    const float a = static_cast<float>(p.tmap[s]) * fr;
    Xs[i] = __float2bfloat16(k < half ? cosf(a) : sinf(a));
  }
  __syncthreads();
  skinny_gemm<MROWS>(Xs, p.n_steps, p.freq, p.t0_w, p.t0_b, H, p.t1, H, EPI_SILU);
  __syncthreads();
  {
    const int rows = bs * T + 1;
    for (int i = tid; i < rows * p.token; i += DS_THREADS) {
      const int r = i / p.token, k = i - r * p.token;
      Xs[i] = r < bs * T ? p.z[static_cast<long long>(r) * p.token + k] : p.uncond[k];
    }
    __syncthreads();
    skinny_gemm<MROWS>(Xs, rows, p.token, p.z_w, p.z_b, H, p.ze, H, EPI_STORE);
  }
  for (int i = tid; i < bs * T * C; i += DS_THREADS) xcur[i] = __bfloat162float(__float2bfloat16(p.noise[i]));
  grid.sync();
  // ---- prologue B: te = W2 t1 + b2
  stage_rows(Xs, p.t1, p.n_steps * H);
  __syncthreads();
  skinny_gemm<MROWS>(Xs, p.n_steps, H, p.t2_w, p.t2_b, H, p.te, H, EPI_STORE);
  grid.sync();

  for (int step = p.n_steps - 1, it = 0; step >= 0; --step, ++it) {
    float* h = (it & 1) ? p.h1 : p.h0;
    // ---- H0: token rows.  row = seq * L + tok; tok < T: te + ze (+ pos); tok >= T: x_embedder(x) (+ pos)
    for (int i = gtid; i < M * H; i += gthreads) {
      const int row = i / H, c = i - row * H;
      const int seq = row / L, tok = row - seq * L;
      const int b = seq < bs ? seq : seq - bs;
      float v;
      if (tok < T) {
        const int zr = seq < bs ? b * T + tok : bs * T;
        v = __ldcg(p.te + step * H + c) + __ldcg(p.ze + zr * H + c);
      } else {
        v = __bfloat162float(p.x_b[c]);
        const float* xr = xcur + (b * T + tok - T) * C;
        for (int k = 0; k < C; ++k)
          v = fmaf(__bfloat162float(__float2bfloat16(xr[k])), __bfloat162float(p.x_w[c * C + k]), v);
      }
      h[i] = v + __bfloat162float(p.pos[tok * H + c]);
    }
    grid.sync();
    for (int l = 0; l < p.depth; ++l) {
      const DitBlockW& w = p.blk[l];
      // ---- P1: qkv = LN(h) Wqkv^T + b
      stage_layernorm(Xs, h, M, H);
      __syncthreads();
      skinny_gemm<MROWS>(Xs, M, H, w.qkv_w, w.qkv_b, 3 * H, p.qkv, 3 * H, EPI_STORE);
      grid.sync();
      // ---- P2: attention (every CTA computes all (sequence, head) pairs: 6x6 scores each) -> O in shared; h += O Wproj^T + b
      {
        bf16* Os = Xs;                                                     // [M][H] bf16
        constexpr float scale = HD == 64 ? 0.125f : 0.10206207261596575f;    // head_dim^-0.5, as the module path's float
        for (int pr = warp; pr < nseq * p.heads; pr += DS_WARPS) {
          const int seq = pr / p.heads, hd = pr - seq * p.heads;
          float2 k[L], v[L];
          float k3[HD == 96 ? L : 1], v3[HD == 96 ? L : 1];           // dims 64..95 (HD = 96 only)
          const float* base = p.qkv + static_cast<long long>(seq * L) * 3 * H + hd * HD + 2 * lane;
          const float* base3 = base + 64 - lane;
#pragma unroll
          for (int i = 0; i < L; ++i) {
            k[i] = __ldcg(reinterpret_cast<const float2*>(base + static_cast<long long>(i) * 3 * H + H));
            v[i] = __ldcg(reinterpret_cast<const float2*>(base + static_cast<long long>(i) * 3 * H + 2 * H));
            if constexpr (HD == 96) {
              k3[i] = __ldcg(base3 + static_cast<long long>(i) * 3 * H + H);
              v3[i] = __ldcg(base3 + static_cast<long long>(i) * 3 * H + 2 * H);
            }
          }
#pragma unroll
          for (int i = 0; i < L; ++i) {                        // one query row at a time: L partial dots, ONE batched butterfly
            const float2 q = __ldcg(reinterpret_cast<const float2*>(base + static_cast<long long>(i) * 3 * H));
            float sc[L];
#pragma unroll
            for (int j = 0; j < L; ++j) sc[j] = q.x * k[j].x + q.y * k[j].y;
            if constexpr (HD == 96) {
              const float q3 = __ldcg(base3 + static_cast<long long>(i) * 3 * H);
#pragma unroll
              for (int j = 0; j < L; ++j) sc[j] = fmaf(q3, k3[j], sc[j]);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1)
#pragma unroll
              for (int j = 0; j < L; ++j) sc[j] += __shfl_xor_sync(0xffffffffu, sc[j], o);
            float mx = -INFINITY;
#pragma unroll
            for (int j = 0; j < L; ++j) mx = fmaxf(mx, sc[j]);
            float den = 0.f, o0 = 0.f, o1 = 0.f, o2 = 0.f;
#pragma unroll
            for (int j = 0; j < L; ++j) {
              const float e = __expf((sc[j] - mx) * scale);
              den += e; o0 = fmaf(e, v[j].x, o0); o1 = fmaf(e, v[j].y, o1);
              if constexpr (HD == 96) o2 = fmaf(e, v3[j], o2);
            }
            const float inv = 1.0f / den;
            *reinterpret_cast<uint32_t*>(Os + (seq * L + i) * H + hd * HD + 2 * lane) = pack_bf16x2(o0 * inv, o1 * inv);
            if constexpr (HD == 96) Os[(seq * L + i) * H + hd * HD + 64 + lane] = __float2bfloat16(o2 * inv);
          }
        }
        __syncthreads();
        skinny_gemm<MROWS>(Os, M, H, w.proj_w, w.proj_b, H, h, H, EPI_ACC);
      }
      grid.sync();
      // ---- P3: u = gelu_tanh(LN(h) Wfc1^T + b)
      stage_layernorm(Xs, h, M, H);
      __syncthreads();
      skinny_gemm<MROWS>(Xs, M, H, w.fc1_w, w.fc1_b, p.mlp, p.u, p.mlp, EPI_GELU);
      grid.sync();
      // ---- P4: h += u Wfc2^T + b
      stage_rows(Xs, p.u, M * p.mlp);
      __syncthreads();
      skinny_gemm<MROWS>(Xs, M, p.mlp, w.fc2_w, w.fc2_b, H, h, H, EPI_ACC);
      grid.sync();
    }
    // ---- final layer on the action rows + guidance + DDIM update: redundantly in every CTA (x stays in shared memory).
    //      h of this step is not written again before two more grid barriers (the next step uses the other h buffer).
    {
      const int arows = nseq * T;
      for (int r = warp; r < arows; r += DS_WARPS) {           // Xs[r][:] = bf16(LN(h[action row r]))
        const int seq = r / T, tok = T + (r - seq * T);
        stage_layernorm_row(Xs + r * H, h + static_cast<long long>(seq * L + tok) * H, H);
      }
      __syncthreads();
      for (int o = warp; o < arows * C; o += DS_WARPS) {       // eps_s[r][cc] = bf16(LN row . fin_w[cc] + fin_b[cc])
        const int r = o / C, cc = o - r * C;
        float s = 0.f;
        for (int c = lane; c < H; c += 32) s = fmaf(__bfloat162float(Xs[r * H + c]), __bfloat162float(p.fin_w[cc * H + c]), s);
        s = warp_sum_f(s);
        if (lane == 0) eps_s[o] = __bfloat162float(__float2bfloat16(s + __bfloat162float(p.fin_b[cc])));
      }
      __syncthreads();
      for (int i = tid; i < bs * T * C; i += DS_THREADS) {
        const int b = i / (T * C), rem = i - b * T * C;
        const float cond = eps_s[b * T * C + rem], unc = eps_s[(bs + b) * T * C + rem];
        const float eps = __bfloat162float(__float2bfloat16(unc + p.cfg_scale * (cond - unc)));     // models.py:262-266
        const float x = xcur[i];
        const float x0 = p.sqrt_recip[step] * x - p.sqrt_recipm1[step] * eps;                       // gaussian_diffusion.py:328,345
        const float e2 = (p.sqrt_recip[step] * x - x0) / p.sqrt_recipm1[step];                      // :554
        const float ab = p.acp_prev[step];
        xcur[i] = x0 * sqrtf(ab) + sqrtf(1.0f - ab) * e2;                                            // :560-565, eta = 0
      }
      __syncthreads();
    }
  }
  if (blockIdx.x == 0)
    for (int i = tid; i < bs * T * C; i += DS_THREADS) p.out[i] = xcur[i];
}

}  // namespace

}  // namespace dvla

using namespace dvla;

extern "C" int dvla_dit_ddim_sample(const dvla_dit_sampler_args* a, void* stream) {
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!a || !a->blocks || !a->z || !a->noise || !a->out || !a->workspace) { set_error("dit_ddim_sample: null pointer"); return DVLA_ERR_INVALID; }
  const int H = (int)a->hidden, T = (int)a->T, C = (int)a->channels, bs = (int)a->batch;
  const int M = 2 * bs * 2 * T;
  const int64_t head_dim = a->heads > 0 && a->hidden % a->heads == 0 ? a->hidden / a->heads : 0;
  if (a->depth <= 0 || a->depth > DS_MAX_DEPTH || a->n_steps <= 0 || a->n_steps > DS_MAX_STEPS || M > DS_MAXM || 2 * T > 8 ||
      (head_dim != 64 && head_dim != 96) || H % 8 || a->token % 8 || a->mlp % 8 || a->freq % 8 || bs * T + 1 > DS_MAXM) {
    set_error("dit_ddim_sample: unsupported shape (rows %d <= %d, tokens per sequence <= 8, head_dim = hidden / heads 64 or 96 "
              "(hidden %lld, heads %lld), dims %% 8)", M, DS_MAXM, (long long)a->hidden, (long long)a->heads);
    return DVLA_ERR_UNSUPPORTED;
  }
  if (dvla_dit_sampler_workspace_bytes(a->batch, a->T, a->hidden, a->mlp, a->n_steps) > a->workspace_bytes) {
    set_error("dit_ddim_sample: workspace too small"); return DVLA_ERR_INVALID;
  }
  DitSamplerParams p;
  memset(&p, 0, sizeof(p));
  for (int l = 0; l < a->depth; ++l) {
    const dvla_dit_block_weights& b = a->blocks[l];
    p.blk[l] = DitBlockW{(const bf16*)b.qkv_w, (const bf16*)b.qkv_b, (const bf16*)b.proj_w, (const bf16*)b.proj_b,
                         (const bf16*)b.fc1_w, (const bf16*)b.fc1_b, (const bf16*)b.fc2_w, (const bf16*)b.fc2_b};
  }
  p.depth = (int)a->depth;
  p.x_w = (const bf16*)a->x_w; p.x_b = (const bf16*)a->x_b; p.t0_w = (const bf16*)a->t0_w; p.t0_b = (const bf16*)a->t0_b;
  p.t2_w = (const bf16*)a->t2_w; p.t2_b = (const bf16*)a->t2_b; p.z_w = (const bf16*)a->z_w; p.z_b = (const bf16*)a->z_b;
  p.uncond = (const bf16*)a->uncondition; p.pos = (const bf16*)a->pos; p.fin_w = (const bf16*)a->final_w; p.fin_b = (const bf16*)a->final_b;
  p.z = (const bf16*)a->z; p.noise = a->noise; p.out = a->out;
  for (int i = 0; i < a->n_steps; ++i) {
    p.tmap[i] = a->timestep_map[i]; p.sqrt_recip[i] = a->sqrt_recip_alphas_cumprod[i];
    p.sqrt_recipm1[i] = a->sqrt_recipm1_alphas_cumprod[i]; p.acp_prev[i] = a->alphas_cumprod_prev[i];
  }
  p.n_steps = (int)a->n_steps; p.cfg_scale = a->cfg_scale;
  p.bs = bs; p.T = T; p.C = C; p.H = H; p.heads = (int)a->heads; p.token = (int)a->token; p.mlp = (int)a->mlp; p.freq = (int)a->freq;
  float* ws = reinterpret_cast<float*>(a->workspace);
  p.h0 = ws; ws += M * H;
  p.h1 = ws; ws += M * H;
  p.qkv = ws; ws += M * 3 * H;
  p.u = ws; ws += M * p.mlp;
  p.te = ws; ws += p.n_steps * H;
  p.t1 = ws; ws += p.n_steps * H;
  p.ze = ws; ws += (bs * T + 1) * H;
  int widest = p.mlp > p.token ? p.mlp : p.token;
  if (p.freq > widest) widest = p.freq;
  int rows = M > bs * T + 1 ? M : bs * T + 1;
  if (p.n_steps > rows) rows = p.n_steps;
  size_t smem = static_cast<size_t>(rows) * widest * 2;
  const size_t xs_bytes = static_cast<size_t>(M) * p.mlp * 2;          // xcur / eps_s sit behind the [M][mlp] staging area
  if (smem < xs_bytes) smem = xs_bytes;
  smem += static_cast<size_t>(bs * T * C + 2 * bs * T * C) * sizeof(float) + 16;
  if (static_cast<size_t>(bs * T + 1) * p.token * 2 > xs_bytes || static_cast<size_t>(p.n_steps) * (p.freq > H ? p.freq : H) * 2 > xs_bytes) {
    set_error("dit_ddim_sample: prologue staging does not fit behind the block staging area"); return DVLA_ERR_UNSUPPORTED;
  }
  if (smem > 227 * 1024) { set_error("dit_ddim_sample: %zu bytes of shared memory needed", smem); return DVLA_ERR_UNSUPPORTED; }
  if (2 * T != 6) { set_error("dit_ddim_sample: built for action_pred_steps == 3 (6 tokens per sequence), got %d", 2 * T); return DVLA_ERR_UNSUPPORTED; }
  void* kern = head_dim == 96 ? reinterpret_cast<void*>(dit_ddim_sample_kernel<12, 6, 96>)
                              : reinterpret_cast<void*>(dit_ddim_sample_kernel<12, 6, 64>);
  static const cudaError_t attr_err64 = cudaFuncSetAttribute(dit_ddim_sample_kernel<12, 6, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  static const cudaError_t attr_err96 = cudaFuncSetAttribute(dit_ddim_sample_kernel<12, 6, 96>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  const cudaError_t attr_err = head_dim == 96 ? attr_err96 : attr_err64;
  if (attr_err != cudaSuccess) { set_error("dit_ddim_sample smem attr: %s", cudaGetErrorString(attr_err)); return DVLA_ERR_CUDA; }
  if (a->n_steps > 12 || bs * T + 1 > 12) { set_error("dit_ddim_sample: prologue rows exceed 12"); return DVLA_ERR_UNSUPPORTED; }
  int dev = 0, coop = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
  if (!coop) { set_error("dit_ddim_sample: device has no cooperative launch"); return DVLA_ERR_UNSUPPORTED; }
  void* args[] = {const_cast<DitSamplerParams*>(&p)};
  cudaError_t e = cudaLaunchCooperativeKernel(kern, dim3(num_sms()), dim3(DS_THREADS), args, smem, s);
  if (e != cudaSuccess) { set_error("dit_ddim_sample launch: %s", cudaGetErrorString(e)); return DVLA_ERR_CUDA; }
  count_launch();
  return DVLA_OK;
}

extern "C" int64_t dvla_dit_sampler_workspace_bytes(int64_t batch, int64_t T, int64_t hidden, int64_t mlp, int64_t n_steps) {
  const int64_t M = 2 * batch * 2 * T;
  return 4 * (2 * M * hidden + M * 3 * hidden + M * mlp + 2 * n_steps * hidden + (batch * T + 1) * hidden);
}
