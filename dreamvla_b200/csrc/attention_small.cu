// Flash attention for SHORT sequences (Lq <= 32, Lk <= 64, head_dim 64 or 96, no mask, no dropout) on the SIMT pipes.
//
// Call site (SURVEY.md 8a): the DiT action head (a-8/a-9: 6 tokens per sequence, 12 blocks, 8*B*S sequences -- reference
// models/action_model/models.py:130-134 via timm Attention).  A 64-row tensor-core tile is 90 % padding for it and one
// (batch, head) per CTA means 7680 CTAs of mostly idle warps; it is latency / launch bound, so the layout is chosen for many
// independent short chains instead:
//   TPR threads per row, DPT = HD / TPR head dims each (one shuffle per thread-count doubling in a dot product), fp32 math,
//   online softmax in the exp2 domain; K / V rows are broadcast reads (all rows of one (batch, head) sit in the same warp
//   or the next).
//     head_dim 64 (DiT-B/L): 2 threads x 32 dims.  head_dim 96 (DiT-S): 4 threads x 24 dims -- with 2 x 48 the dK/dV kernel
//     would keep 6 x 48 = 288 floats live per thread, more than the 255 registers a thread can have.
//   forward:   thread group = one query row, loop over keys
//   backward:  dQ: thread group = one query row (also writes delta = rowsum(dO * O)); dK/dV: thread group = one KEY row,
//              loop over the <= 32 queries with the stored LSE -- no atomics.
#include "common.cuh"
#include "host.cuh"
#include "../../include/dvla.h"

namespace dvla {
namespace {

constexpr float SM_LOG2E = 1.4426950408889634f;
constexpr float SM_LN2 = 0.6931471805599453f;

struct SmallParams {
  const bf16 *q, *k, *v, *o, *d_o;
  bf16 *out, *dq, *dk, *dv;
  float* lse;
  float* delta;
  const float* key_bias;        // optional [Lk], natural-log units
  int B, H, Lq, Lk;
  long long q_sb, q_ss, q_sh, k_sb, k_ss, k_sh, v_sb, v_ss, v_sh, o_sb, o_ss, o_sh;
  long long do_sb, do_ss, do_sh, dq_sb, dq_ss, dq_sh, dk_sb, dk_ss, dk_sh, dv_sb, dv_ss, dv_sh;
  float scale;
};

template <int N>    // N bf16 (N % 8 == 0, 16-byte aligned) -> fp32
__device__ __forceinline__ void load_part(const bf16* p, float (&f)[N]) {
#pragma unroll
  for (int i = 0; i < N / 8; ++i) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(p) + i);
    float2 t;
    t = unpack_bf16x2(u.x); f[i * 8 + 0] = t.x; f[i * 8 + 1] = t.y;
    t = unpack_bf16x2(u.y); f[i * 8 + 2] = t.x; f[i * 8 + 3] = t.y;
    t = unpack_bf16x2(u.z); f[i * 8 + 4] = t.x; f[i * 8 + 5] = t.y;
    t = unpack_bf16x2(u.w); f[i * 8 + 6] = t.x; f[i * 8 + 7] = t.y;
  }
}
template <int N>
__device__ __forceinline__ void store_part(bf16* p, const float (&f)[N], float mul) {
#pragma unroll
  for (int i = 0; i < N / 8; ++i)
    reinterpret_cast<uint4*>(p)[i] = make_uint4(pack_bf16x2(f[i * 8 + 0] * mul, f[i * 8 + 1] * mul), pack_bf16x2(f[i * 8 + 2] * mul, f[i * 8 + 3] * mul),
                                                pack_bf16x2(f[i * 8 + 4] * mul, f[i * 8 + 5] * mul), pack_bf16x2(f[i * 8 + 6] * mul, f[i * 8 + 7] * mul));
}
template <int TPR, int N>
__device__ __forceinline__ float dot_part(const float (&a)[N], const float (&b)[N]) {
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
  for (int i = 0; i < N; i += 4) {
    s0 = fmaf(a[i], b[i], s0); s1 = fmaf(a[i + 1], b[i + 1], s1); s2 = fmaf(a[i + 2], b[i + 2], s2); s3 = fmaf(a[i + 3], b[i + 3], s3);
  }
  float s = (s0 + s1) + (s2 + s3);
#pragma unroll
  for (int o = 1; o < TPR; o <<= 1) s = s + __shfl_xor_sync(0xffffffffu, s, o);   // the row's other threads hold the other dims
  return s;
}

// Threads per row for a head dim: 2 x 32 dims at 64, 4 x 24 dims at 96 (both: whole 16-byte chunks per thread).
template <int HD> struct SmallLayout;
template <> struct SmallLayout<64> { static constexpr int TPR = 2, LOG2_TPR = 1; };
template <> struct SmallLayout<96> { static constexpr int TPR = 4, LOG2_TPR = 2; };

// thread group [TPR*r, TPR*r + TPR) <-> row r of the flattened (b, h, i) index; a group is always active together
// (TPR divides 32)
template <int HD>
__global__ void __launch_bounds__(256) attn_small_fwd_kernel(const SmallParams p) {
  constexpr int TPR = SmallLayout<HD>::TPR, DPT = HD / TPR;
  const long long gid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long rowid = gid >> SmallLayout<HD>::LOG2_TPR;
  const int part = static_cast<int>(gid & (TPR - 1));
  const long long total = static_cast<long long>(p.B) * p.H * p.Lq;
  const bool live = rowid < total;
  const long long rid = live ? rowid : total - 1;       // dead threads shadow the last row (keeps shuffles convergent)
  const int i = static_cast<int>(rid % p.Lq);
  const int h = static_cast<int>((rid / p.Lq) % p.H);
  const int b = static_cast<int>(rid / (static_cast<long long>(p.Lq) * p.H));
  float q[DPT], acc[DPT];
  load_part(p.q + b * p.q_sb + static_cast<long long>(i) * p.q_ss + h * p.q_sh + part * DPT, q);
#pragma unroll
  for (int d = 0; d < DPT; ++d) acc[d] = 0.f;
  const float sc = p.scale * SM_LOG2E;
  float m = -INFINITY, l = 0.f;
  const bf16* kp = p.k + b * p.k_sb + h * p.k_sh + part * DPT;
  const bf16* vp = p.v + b * p.v_sb + h * p.v_sh + part * DPT;
  for (int j = 0; j < p.Lk; ++j) {
    float kk[DPT], vv[DPT];
    load_part(kp + static_cast<long long>(j) * p.k_ss, kk);
    load_part(vp + static_cast<long long>(j) * p.v_ss, vv);
    const float s = dot_part<TPR>(q, kk) * sc + (p.key_bias ? __ldg(p.key_bias + j) * SM_LOG2E : 0.f);
    const float m_new = fmaxf(m, s);
    const float corr = ex2_approx(m - m_new);           // m = -inf on the first key -> 0
    const float e = ex2_approx(s - m_new);
    l = l * corr + e;
#pragma unroll
    for (int d = 0; d < DPT; ++d) acc[d] = fmaf(acc[d], corr, e * vv[d]);
    m = m_new;
  }
  if (live) {
    store_part(p.out + b * p.o_sb + static_cast<long long>(i) * p.o_ss + h * p.o_sh + part * DPT, acc, 1.0f / l);
    if (p.lse && part == 0) p.lse[rid] = (m + log2f(l)) * SM_LN2;
  }
}

template <int HD>
__global__ void __launch_bounds__(256) attn_small_bwd_dq_kernel(const SmallParams p) {
  constexpr int TPR = SmallLayout<HD>::TPR, DPT = HD / TPR;
  const long long gid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long rowid = gid >> SmallLayout<HD>::LOG2_TPR;
  const int part = static_cast<int>(gid & (TPR - 1));
  const long long total = static_cast<long long>(p.B) * p.H * p.Lq;
  const bool live = rowid < total;
  const long long rid = live ? rowid : total - 1;
  const int i = static_cast<int>(rid % p.Lq);
  const int h = static_cast<int>((rid / p.Lq) % p.H);
  const int b = static_cast<int>(rid / (static_cast<long long>(p.Lq) * p.H));
  float q[DPT], g[DPT], acc[DPT];
  load_part(p.q + b * p.q_sb + static_cast<long long>(i) * p.q_ss + h * p.q_sh + part * DPT, q);
  load_part(p.d_o + b * p.do_sb + static_cast<long long>(i) * p.do_ss + h * p.do_sh + part * DPT, g);
  {
    float o[DPT];
    load_part(p.o + b * p.o_sb + static_cast<long long>(i) * p.o_ss + h * p.o_sh + part * DPT, o);
    const float dl = dot_part<TPR>(o, g);                    // delta_i = sum_d dO * O  (FlashAttention-2 backward)
    if (live && part == 0) p.delta[rid] = dl;
#pragma unroll
    for (int d = 0; d < DPT; ++d) acc[d] = 0.f;
    const float sc = p.scale * SM_LOG2E;
    const float lse2 = p.lse[rid] * SM_LOG2E;
    const bf16* kp = p.k + b * p.k_sb + h * p.k_sh + part * DPT;
    const bf16* vp = p.v + b * p.v_sb + h * p.v_sh + part * DPT;
    for (int j = 0; j < p.Lk; ++j) {
      float kk[DPT], vv[DPT];
      load_part(kp + static_cast<long long>(j) * p.k_ss, kk);
      load_part(vp + static_cast<long long>(j) * p.v_ss, vv);
      const float pr = ex2_approx(dot_part<TPR>(q, kk) * sc + (p.key_bias ? __ldg(p.key_bias + j) * SM_LOG2E : 0.f) - lse2);
      const float ds = pr * (dot_part<TPR>(g, vv) - dl);
#pragma unroll
      for (int d = 0; d < DPT; ++d) acc[d] = fmaf(ds, kk[d], acc[d]);
    }
  }
  if (live) store_part(p.dq + b * p.dq_sb + static_cast<long long>(i) * p.dq_ss + h * p.dq_sh + part * DPT, acc, p.scale);
}

// thread group <-> KEY row j of (b, h); needs delta (written by the dQ kernel launched before it on the same stream)
template <int HD>
__global__ void __launch_bounds__(256) attn_small_bwd_dkv_kernel(const SmallParams p) {
  constexpr int TPR = SmallLayout<HD>::TPR, DPT = HD / TPR;
  const long long gid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long rowid = gid >> SmallLayout<HD>::LOG2_TPR;
  const int part = static_cast<int>(gid & (TPR - 1));
  const long long total = static_cast<long long>(p.B) * p.H * p.Lk;
  const bool live = rowid < total;
  const long long rid = live ? rowid : total - 1;
  const int j = static_cast<int>(rid % p.Lk);
  const int h = static_cast<int>((rid / p.Lk) % p.H);
  const int b = static_cast<int>(rid / (static_cast<long long>(p.Lk) * p.H));
  float kk[DPT], vv[DPT], dk[DPT], dv[DPT];
  load_part(p.k + b * p.k_sb + static_cast<long long>(j) * p.k_ss + h * p.k_sh + part * DPT, kk);
  load_part(p.v + b * p.v_sb + static_cast<long long>(j) * p.v_ss + h * p.v_sh + part * DPT, vv);
#pragma unroll
  for (int d = 0; d < DPT; ++d) { dk[d] = 0.f; dv[d] = 0.f; }
  const float sc = p.scale * SM_LOG2E;
  const float kb = p.key_bias ? __ldg(p.key_bias + j) * SM_LOG2E : 0.f;
  const long long bh = static_cast<long long>(b) * p.H + h;
  const bf16* qp = p.q + b * p.q_sb + h * p.q_sh + part * DPT;
  const bf16* gp = p.d_o + b * p.do_sb + h * p.do_sh + part * DPT;
  for (int i = 0; i < p.Lq; ++i) {
    float q[DPT], g[DPT];
    load_part(qp + static_cast<long long>(i) * p.q_ss, q);
    load_part(gp + static_cast<long long>(i) * p.do_ss, g);
    const float pr = ex2_approx(dot_part<TPR>(q, kk) * sc + kb - __ldg(p.lse + bh * p.Lq + i) * SM_LOG2E);
    const float ds = pr * (dot_part<TPR>(g, vv) - __ldg(p.delta + bh * p.Lq + i));
#pragma unroll
    for (int d = 0; d < DPT; ++d) { dv[d] = fmaf(pr, g[d], dv[d]); dk[d] = fmaf(ds, q[d], dk[d]); }
  }
  if (live) {
    store_part(p.dk + b * p.dk_sb + static_cast<long long>(j) * p.dk_ss + h * p.dk_sh + part * DPT, dk, p.scale);
    store_part(p.dv + b * p.dv_sb + static_cast<long long>(j) * p.dv_ss + h * p.dv_sh + part * DPT, dv, 1.0f);
  }
}

// The SmallParams fields the forward and backward share: operands q/k/v and lse, dims, strides, scale and key bias.
template <class Args>
SmallParams small_params(const Args* a) {
  SmallParams p{};
  p.q = (const bf16*)a->q; p.k = (const bf16*)a->k; p.v = (const bf16*)a->v; p.lse = const_cast<float*>(a->lse);
  p.B = (int)a->B; p.H = (int)a->H; p.Lq = (int)a->Lq; p.Lk = (int)a->Lk; p.scale = a->scale; p.key_bias = a->key_bias;
  p.q_sb = a->q_sb; p.q_ss = a->q_ss; p.q_sh = a->q_sh; p.k_sb = a->k_sb; p.k_ss = a->k_ss; p.k_sh = a->k_sh;
  p.v_sb = a->v_sb; p.v_ss = a->v_ss; p.v_sh = a->v_sh; p.o_sb = a->o_sb; p.o_ss = a->o_ss; p.o_sh = a->o_sh;
  return p;
}

}  // namespace

// The serial key loop of these row kernels loses to the mma.sync kernel once there are hundreds of keys per row, so they
// take the short-key case only (the DiT blocks: 6 x 6 per (b,h)).
constexpr int SMALL_MAX_LQ = 32;
constexpr int SMALL_MAX_LK = 64;

bool attn_small_applicable(int64_t Lq, int64_t Lk, const void* mask, float dropout_p) {
  return Lq <= SMALL_MAX_LQ && Lk <= SMALL_MAX_LK && !mask && dropout_p == 0.f;
}

template <int HD>
static int small_fwd_launch(const SmallParams& p, const dvla_attn_fwd_args* a, cudaStream_t s) {
  const long long threads = SmallLayout<HD>::TPR * a->B * a->H * a->Lq;
  attn_small_fwd_kernel<HD><<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(p);
  DVLA_CHECK_LAUNCH("attn_small_fwd");
  return DVLA_OK;
}

template <int HD>
static int small_bwd_launch(const SmallParams& p, const dvla_attn_bwd_args* a, cudaStream_t s) {
  const long long tq = SmallLayout<HD>::TPR * a->B * a->H * a->Lq, tk = SmallLayout<HD>::TPR * a->B * a->H * a->Lk;
  attn_small_bwd_dq_kernel<HD><<<(unsigned)((tq + 255) / 256), 256, 0, s>>>(p);
  DVLA_CHECK_LAUNCH("attn_small_bwd_dq");
  attn_small_bwd_dkv_kernel<HD><<<(unsigned)((tk + 255) / 256), 256, 0, s>>>(p);
  DVLA_CHECK_LAUNCH("attn_small_bwd_dkv");
  return DVLA_OK;
}

// a->head_dim is 0, 64 or 96 here (checked by dvla_attn_fwd / dvla_attn_bwd before they dispatch)
int attn_small_fwd(const dvla_attn_fwd_args* a, cudaStream_t s) {
  SmallParams p = small_params(a);
  p.out = (bf16*)a->o;
  return a->head_dim == 96 ? small_fwd_launch<96>(p, a, s) : small_fwd_launch<64>(p, a, s);
}

int attn_small_bwd(const dvla_attn_bwd_args* a, cudaStream_t s) {
  SmallParams p = small_params(a);
  p.o = (const bf16*)a->o; p.d_o = (const bf16*)a->d_o; p.dq = (bf16*)a->dq; p.dk = (bf16*)a->dk; p.dv = (bf16*)a->dv;
  p.delta = a->delta;
  p.do_sb = a->do_sb; p.do_ss = a->do_ss; p.do_sh = a->do_sh;
  p.dq_sb = a->dq_sb; p.dq_ss = a->dq_ss; p.dq_sh = a->dq_sh; p.dk_sb = a->dk_sb; p.dk_ss = a->dk_ss; p.dk_sh = a->dk_sh;
  p.dv_sb = a->dv_sb; p.dv_ss = a->dv_ss; p.dv_sh = a->dv_sh;
  return a->head_dim == 96 ? small_bwd_launch<96>(p, a, s) : small_bwd_launch<64>(p, a, s);
}

}  // namespace dvla
