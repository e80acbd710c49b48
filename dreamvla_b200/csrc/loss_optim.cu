// Fused loss kernels (value + gradient in one pass) and the flat-buffer optimiser (grad-norm, clip, AdamW).
// All HBM-bound: 16-byte vector accesses, grid-stride loops sized against the SM count, block reduce -> one atomicAdd.
#include "common.cuh"
#include "../../include/dvla.h"

namespace dvla {
void set_error(const char* fmt, ...);
void count_launch();
int num_sms();

#define DVLA_CHECK_LAUNCH(name)                                                                 \
  do {                                                                                          \
    cudaError_t e__ = cudaGetLastError();                                                       \
    if (e__ != cudaSuccess) { set_error("%s launch: %s", name, cudaGetErrorString(e__)); return DVLA_ERR_CUDA; } \
    count_launch();                                                                             \
  } while (0)

__device__ __forceinline__ float block_sum_256(float v) {
  __shared__ float red[8];
  __syncthreads();
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = (threadIdx.x < 8) ? red[threadIdx.x] : 0.f;
  if (threadIdx.x < 32) t = warp_sum(t);
  return t;  // valid in warp 0
}

static inline unsigned grid_for(long long work_items, int per_block) {
  long long b = (work_items + per_block - 1) / per_block;
  const long long cap = 8LL * num_sms();
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (unsigned)b;
}

// ---------------------------------------------------------------------------------------------------------------
// MSE with optional per-row {0,1} mask:  mean((pred*m - label*m)^2) over rows*C   (train_utils.py:325-337, 499-502)
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) mse_loss_kernel(const bf16* __restrict__ pred, const bf16* __restrict__ label,
                                                       const float* __restrict__ row_mask, long long rows, int C,
                                                       float weight, float* __restrict__ loss_out,
                                                       bf16* __restrict__ dpred) {
  const long long total = rows * C;
  const float inv = 1.0f / static_cast<float>(total);
  float acc = 0.f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float m = row_mask ? row_mask[i / C] : 1.0f;
    const float d = (__bfloat162float(pred[i]) - __bfloat162float(label[i])) * m;
    acc += d * d;
    if (dpred) dpred[i] = __float2bfloat16(weight * 2.0f * d * m * inv);
  }
  const float t = block_sum_256(acc);
  if (threadIdx.x == 0) atomicAdd(loss_out, weight * t * inv);
}
int mse_loss_dispatch(const void* pred, const void* label, const float* row_mask, int64_t rows, int64_t C, float weight,
                      float* loss_out, void* dpred, cudaStream_t s) {
  if (!pred || !label || !loss_out) { set_error("mse_loss: null pointer"); return DVLA_ERR_INVALID; }
  if (rows <= 0 || C <= 0) return DVLA_OK;
  mse_loss_kernel<<<grid_for(rows * C, 256 * 8), 256, 0, s>>>((const bf16*)pred, (const bf16*)label, row_mask, rows,
                                                             (int)C, weight, loss_out, (bf16*)dpred);
  DVLA_CHECK_LAUNCH("mse_loss");
  return DVLA_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// mean_rows(1 - cos(pred_row, label_row))   (train_utils.py:423-425, 448-450; F.cosine_similarity eps = 1e-8)
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) cosine_loss_kernel(const bf16* __restrict__ pred, const bf16* __restrict__ label,
                                                          long long rows, int C, float weight,
                                                          float* __restrict__ loss_out, bf16* __restrict__ dpred) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float acc = 0.f;
  const float invr = 1.0f / static_cast<float>(rows);
  for (long long row = static_cast<long long>(blockIdx.x) * 8 + warp; row < rows; row += static_cast<long long>(gridDim.x) * 8) {
    const bf16* p = pred + row * C;
    const bf16* l = label + row * C;
    float pl = 0.f, pp = 0.f, ll = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float a = __bfloat162float(p[c]), b = __bfloat162float(l[c]);
      pl += a * b; pp += a * a; ll += b * b;
    }
    pl = warp_sum(pl); pp = warp_sum(pp); ll = warp_sum(ll);
    const float np = fmaxf(sqrtf(pp), 1e-8f), nl = fmaxf(sqrtf(ll), 1e-8f);
    const float cosv = pl / (np * nl);
    if (lane == 0) acc += 1.0f - cosv;
    if (dpred) {
      // d(1-cos)/dp = -( l/(np*nl) - cos * p / np^2 )
      const float k1 = 1.0f / (np * nl), k2 = cosv / (np * np);
      bf16* d = dpred + row * C;
      for (int c = lane; c < C; c += 32) {
        const float a = __bfloat162float(p[c]), b = __bfloat162float(l[c]);
        d[c] = __float2bfloat16(-weight * invr * (b * k1 - a * k2));
      }
    }
  }
  const float t = block_sum_256(acc);
  if (threadIdx.x == 0) atomicAdd(loss_out, weight * t * invr);
}
int cosine_loss_dispatch(const void* pred, const void* label, int64_t rows, int64_t C, float weight, float* loss_out,
                         void* dpred, cudaStream_t s) {
  if (!pred || !label || !loss_out) { set_error("cosine_loss: null pointer"); return DVLA_ERR_INVALID; }
  if (rows <= 0 || C <= 0) return DVLA_OK;
  cosine_loss_kernel<<<grid_for(rows, 8), 256, 0, s>>>((const bf16*)pred, (const bf16*)label, rows, (int)C, weight,
                                                      loss_out, (bf16*)dpred);
  DVLA_CHECK_LAUNCH("cosine_loss");
  return DVLA_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Scale-invariant log loss (utils/sigloss.py:11-15): d = log(t+1e-6) - log(p+1e-6); sqrt(mean(d^2) - lambd*mean(d)^2)
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) silog_stats_kernel(const bf16* __restrict__ pred, const bf16* __restrict__ label,
                                                          long long n, float* __restrict__ stats) {
  float s1 = 0.f, s2 = 0.f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float d = logf(__bfloat162float(label[i]) + 1e-6f) - logf(__bfloat162float(pred[i]) + 1e-6f);
    s1 += d; s2 += d * d;
  }
  const float t1 = block_sum_256(s1);
  const float t2 = block_sum_256(s2);
  if (threadIdx.x == 0) { atomicAdd(stats, t1); atomicAdd(stats + 1, t2); }
}
__global__ void __launch_bounds__(256) silog_finish_kernel(const bf16* __restrict__ pred, const bf16* __restrict__ label,
                                                           long long n, const float* __restrict__ stats, float lambd,
                                                           float weight, float* __restrict__ loss_out,
                                                           bf16* __restrict__ dpred) {
  const float invn = 1.0f / static_cast<float>(n);
  const float md = stats[0] * invn, md2 = stats[1] * invn;
  const float loss = sqrtf(fmaxf(md2 - lambd * md * md, 0.f));
  if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(loss_out, weight * loss);
  if (!dpred) return;
  const float k = weight / (2.0f * fmaxf(loss, 1e-12f));
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float pv = __bfloat162float(pred[i]) + 1e-6f;
    const float d = logf(__bfloat162float(label[i]) + 1e-6f) - logf(pv);
    // dL/dd_i = (2 d_i - 2 lambd md)/n / (2L);  dd_i/dp_i = -1/(p_i+1e-6)
    dpred[i] = __float2bfloat16(-k * (2.0f * d - 2.0f * lambd * md) * invn / pv);
  }
}
int silog_stats_dispatch(const void* pred, const void* label, int64_t n, float* stats, cudaStream_t s) {
  if (!pred || !label || !stats) { set_error("silog_stats: null pointer"); return DVLA_ERR_INVALID; }
  if (n <= 0) return DVLA_OK;
  silog_stats_kernel<<<grid_for(n, 256 * 8), 256, 0, s>>>((const bf16*)pred, (const bf16*)label, n, stats);
  DVLA_CHECK_LAUNCH("silog_stats");
  return DVLA_OK;
}
int silog_finish_dispatch(const void* pred, const void* label, int64_t n, const float* stats, float lambd, float weight,
                          float* loss_out, void* dpred, cudaStream_t s) {
  if (!pred || !label || !stats || !loss_out) { set_error("silog_finish: null pointer"); return DVLA_ERR_INVALID; }
  if (n <= 0) return DVLA_OK;
  silog_finish_kernel<<<grid_for(n, 256 * 8), 256, 0, s>>>((const bf16*)pred, (const bf16*)label, n, stats, lambd, weight,
                                                          loss_out, (bf16*)dpred);
  DVLA_CHECK_LAUNCH("silog_finish");
  return DVLA_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Optimiser
// ---------------------------------------------------------------------------------------------------------------
// Global gradient norm.  The result feeds the clip factor of every data-parallel replica, so it must be BIT-identical on
// all ranks for identical (all-reduced) gradients: block partials go to a scratch array and the last block to finish
// (ticket counter) adds them in a fixed order -- no floating-point atomics, no dependence on block scheduling.
constexpr int SUMSQ_MAX_BLOCKS = 2048;
__device__ float g_sumsq_partials[SUMSQ_MAX_BLOCKS];
__device__ unsigned int g_sumsq_ticket = 0;

__global__ void __launch_bounds__(256) sumsq_kernel(const bf16* __restrict__ g, long long n, float* __restrict__ out) {
  float acc = 0.f;
  const long long nv = n >> 3;
  const uint4* gv = reinterpret_cast<const uint4*>(g);
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint4 u = gv[i];
    float2 t;
    t = unpack_bf16x2(u.x); acc += t.x * t.x + t.y * t.y;
    t = unpack_bf16x2(u.y); acc += t.x * t.x + t.y * t.y;
    t = unpack_bf16x2(u.z); acc += t.x * t.x + t.y * t.y;
    t = unpack_bf16x2(u.w); acc += t.x * t.x + t.y * t.y;
  }
  if (blockIdx.x == 0)
    for (long long i = (nv << 3) + threadIdx.x; i < n; i += blockDim.x) { const float f = __bfloat162float(g[i]); acc += f * f; }
  const float t = block_sum_256(acc);
  __shared__ bool s_last;
  if (threadIdx.x == 0) {
    g_sumsq_partials[blockIdx.x] = t;
    __threadfence();
    s_last = atomicAdd(&g_sumsq_ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (s_last) {
    __threadfence();
    float a = 0.f;
    for (unsigned i = threadIdx.x; i < gridDim.x; i += 256) a += __ldcg(&g_sumsq_partials[i]);
    const float total = block_sum_256(a);
    if (threadIdx.x == 0) {
      out[0] += total;
      g_sumsq_ticket = 0;
    }
  }
}
int sumsq_dispatch(const void* g, int64_t n, float* out, cudaStream_t s) {
  if (!g || !out) { set_error("sumsq: null pointer"); return DVLA_ERR_INVALID; }
  if (reinterpret_cast<uintptr_t>(g) & 15) { set_error("sumsq: buffer must be 16-byte aligned"); return DVLA_ERR_INVALID; }
  if (n <= 0) return DVLA_OK;
  unsigned blocks = grid_for(n, 256 * 8 * 4);
  if (blocks > SUMSQ_MAX_BLOCKS) blocks = SUMSQ_MAX_BLOCKS;
  sumsq_kernel<<<blocks, 256, 0, s>>>((const bf16*)g, n, out);
  DVLA_CHECK_LAUNCH("sumsq");
  return DVLA_OK;
}

// In-place clip of the (rank-summed) accumulated gradient: g *= grad_scale * min(1, max_norm / (||g||*grad_scale + 1e-6)).
// Reference utils/train_utils.py:599-600 clips the ACCUMULATED gradient after every micro-step; with gradient accumulation
// that clip must land in the buffer itself (the fused clip inside adamw_kernel only covers accumulation == 1).
__global__ void __launch_bounds__(256) grad_clip_scale_kernel(bf16* __restrict__ g, long long n, const float* __restrict__ sumsq,
                                                              float max_norm, float grad_scale) {
  const float norm = sqrtf(sumsq[0]) * grad_scale;
  const float c = grad_scale * fminf(1.0f, max_norm / (norm + 1e-6f));
  if (c == 1.0f) return;
  const long long nv = n >> 3;
  uint4* gv = reinterpret_cast<uint4*>(g);
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    uint4 u = gv[i];
    float2 t;
    t = unpack_bf16x2(u.x); u.x = pack_bf16x2(t.x * c, t.y * c);
    t = unpack_bf16x2(u.y); u.y = pack_bf16x2(t.x * c, t.y * c);
    t = unpack_bf16x2(u.z); u.z = pack_bf16x2(t.x * c, t.y * c);
    t = unpack_bf16x2(u.w); u.w = pack_bf16x2(t.x * c, t.y * c);
    gv[i] = u;
  }
  if (blockIdx.x == 0)
    for (long long i = (nv << 3) + threadIdx.x; i < n; i += blockDim.x) g[i] = __float2bfloat16(__bfloat162float(g[i]) * c);
}
int grad_clip_scale_dispatch(void* g, int64_t n, const float* sumsq, float max_norm, float grad_scale, cudaStream_t s) {
  if (!g || !sumsq) { set_error("grad_clip_scale: null pointer"); return DVLA_ERR_INVALID; }
  if (reinterpret_cast<uintptr_t>(g) & 15) { set_error("grad_clip_scale: buffer must be 16-byte aligned"); return DVLA_ERR_INVALID; }
  if (n <= 0) return DVLA_OK;
  grad_clip_scale_kernel<<<grid_for(n, 256 * 8 * 4), 256, 0, s>>>((bf16*)g, n, sumsq, max_norm, grad_scale);
  DVLA_CHECK_LAUNCH("grad_clip_scale");
  return DVLA_OK;
}

struct AdamWParams {
  bf16* p; bf16* g; float* m; float* v; long long n;
  const float* sumsq; const float* lr; const float* step;
  float beta1, beta2, eps, wd, max_norm, grad_scale; int zero_grad;
};
__global__ void __launch_bounds__(256) adamw_kernel(AdamWParams a) {
  float clip = a.grad_scale;
  if (a.sumsq) {
    const float norm = sqrtf(a.sumsq[0]) * a.grad_scale;
    clip *= fminf(1.0f, a.max_norm / (norm + 1e-6f));  // torch.nn.utils.clip_grad_norm_ semantics
  }
  const float lr = a.lr[0];
  const float t = a.step[0];
  const float bc1 = 1.0f - powf(a.beta1, t);
  const float bc2s = sqrtf(1.0f - powf(a.beta2, t));
  const float step_size = lr / bc1;
  const float decay = 1.0f - lr * a.wd;
  const long long nv = a.n >> 3;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    uint4 pu = reinterpret_cast<uint4*>(a.p)[i];
    const uint4 gu = reinterpret_cast<const uint4*>(a.g)[i];
    float4 m0 = reinterpret_cast<float4*>(a.m)[2 * i], m1 = reinterpret_cast<float4*>(a.m)[2 * i + 1];
    float4 v0 = reinterpret_cast<float4*>(a.v)[2 * i], v1 = reinterpret_cast<float4*>(a.v)[2 * i + 1];
    float pf[8], gf[8], mf[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w},
                        vf[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
    float2 f;
    f = unpack_bf16x2(pu.x); pf[0] = f.x; pf[1] = f.y; f = unpack_bf16x2(pu.y); pf[2] = f.x; pf[3] = f.y;
    f = unpack_bf16x2(pu.z); pf[4] = f.x; pf[5] = f.y; f = unpack_bf16x2(pu.w); pf[6] = f.x; pf[7] = f.y;
    f = unpack_bf16x2(gu.x); gf[0] = f.x; gf[1] = f.y; f = unpack_bf16x2(gu.y); gf[2] = f.x; gf[3] = f.y;
    f = unpack_bf16x2(gu.z); gf[4] = f.x; gf[5] = f.y; f = unpack_bf16x2(gu.w); gf[6] = f.x; gf[7] = f.y;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float gj = gf[j] * clip;
      mf[j] = a.beta1 * mf[j] + (1.0f - a.beta1) * gj;
      vf[j] = a.beta2 * vf[j] + (1.0f - a.beta2) * gj * gj;
      const float denom = sqrtf(vf[j]) / bc2s + a.eps;
      pf[j] = pf[j] * decay - step_size * mf[j] / denom;
    }
    pu = make_uint4(pack_bf16x2(pf[0], pf[1]), pack_bf16x2(pf[2], pf[3]), pack_bf16x2(pf[4], pf[5]), pack_bf16x2(pf[6], pf[7]));
    reinterpret_cast<uint4*>(a.p)[i] = pu;
    reinterpret_cast<float4*>(a.m)[2 * i] = make_float4(mf[0], mf[1], mf[2], mf[3]);
    reinterpret_cast<float4*>(a.m)[2 * i + 1] = make_float4(mf[4], mf[5], mf[6], mf[7]);
    reinterpret_cast<float4*>(a.v)[2 * i] = make_float4(vf[0], vf[1], vf[2], vf[3]);
    reinterpret_cast<float4*>(a.v)[2 * i + 1] = make_float4(vf[4], vf[5], vf[6], vf[7]);
    if (a.zero_grad) reinterpret_cast<uint4*>(a.g)[i] = make_uint4(0, 0, 0, 0);
  }
  if (blockIdx.x == 0) {
    for (long long i = (nv << 3) + threadIdx.x; i < a.n; i += blockDim.x) {
      const float gj = __bfloat162float(a.g[i]) * clip;
      const float mj = a.beta1 * a.m[i] + (1.0f - a.beta1) * gj;
      const float vj = a.beta2 * a.v[i] + (1.0f - a.beta2) * gj * gj;
      a.m[i] = mj; a.v[i] = vj;
      const float denom = sqrtf(vj) / bc2s + a.eps;
      a.p[i] = __float2bfloat16(__bfloat162float(a.p[i]) * decay - step_size * mj / denom);
      if (a.zero_grad) a.g[i] = __float2bfloat16(0.f);
    }
  }
}
int adamw_dispatch(const dvla_adamw_args* a, cudaStream_t s) {
  if (!a || !a->p || !a->g || !a->m || !a->v || !a->lr || !a->step) { set_error("adamw: null pointer"); return DVLA_ERR_INVALID; }
  if ((reinterpret_cast<uintptr_t>(a->p) | reinterpret_cast<uintptr_t>(a->g) | reinterpret_cast<uintptr_t>(a->m) |
       reinterpret_cast<uintptr_t>(a->v)) & 15) { set_error("adamw: buffers must be 16-byte aligned"); return DVLA_ERR_INVALID; }
  if (a->n <= 0) return DVLA_OK;
  AdamWParams k{(bf16*)a->p, (bf16*)a->g, a->m, a->v, a->n, a->sumsq, a->lr, a->step,
                a->beta1, a->beta2, a->eps, a->weight_decay, a->max_norm, a->grad_scale, a->zero_grad};
  adamw_kernel<<<grid_for(a->n, 256 * 8 * 2), 256, 0, s>>>(k);
  DVLA_CHECK_LAUNCH("adamw");
  return DVLA_OK;
}

// The same clip + AdamW on fp32 master weights: the update lands in p32 (no bf16 rounding of the parameter between
// steps), then the bf16 working copy the kernels read is written as round-to-nearest(p32).  Same formula and operation
// order as adamw_kernel, except that the decay product p * (1 - lr*wd) is rounded on its own (__fmul_rn, no FMA with the
// update), as torch.optim.AdamW's `param.mul_(1 - lr * wd)` does: at lr*wd ~ 1e-7 the decay is about one fp32 ulp of the
// weight, and folding its rounding into the update's drifts the fp32 trajectory by ~6e-4 of the accumulated update over
// 100 steps (2.5e-6 with the separate rounding).  The old bf16 copy is never read.  30 B per parameter (adamw_kernel: 24).
struct AdamWMasterParams {
  float* p32; bf16* p; bf16* g; float* m; float* v; long long n;
  const float* sumsq; const float* lr; const float* step;
  float beta1, beta2, eps, wd, max_norm, grad_scale; int zero_grad;
};
__global__ void __launch_bounds__(256) adamw_master_kernel(AdamWMasterParams a) {
  float clip = a.grad_scale;
  if (a.sumsq) {
    const float norm = sqrtf(a.sumsq[0]) * a.grad_scale;
    clip *= fminf(1.0f, a.max_norm / (norm + 1e-6f));  // torch.nn.utils.clip_grad_norm_ semantics
  }
  const float lr = a.lr[0];
  const float t = a.step[0];
  const float bc1 = 1.0f - powf(a.beta1, t);
  const float bc2s = sqrtf(1.0f - powf(a.beta2, t));
  const float step_size = lr / bc1;
  const float decay = 1.0f - lr * a.wd;
  const long long nv = a.n >> 3;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint4 gu = reinterpret_cast<const uint4*>(a.g)[i];
    float4 p0 = reinterpret_cast<float4*>(a.p32)[2 * i], p1 = reinterpret_cast<float4*>(a.p32)[2 * i + 1];
    float4 m0 = reinterpret_cast<float4*>(a.m)[2 * i], m1 = reinterpret_cast<float4*>(a.m)[2 * i + 1];
    float4 v0 = reinterpret_cast<float4*>(a.v)[2 * i], v1 = reinterpret_cast<float4*>(a.v)[2 * i + 1];
    float pf[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w}, gf[8],
          mf[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w}, vf[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
    float2 f;
    f = unpack_bf16x2(gu.x); gf[0] = f.x; gf[1] = f.y; f = unpack_bf16x2(gu.y); gf[2] = f.x; gf[3] = f.y;
    f = unpack_bf16x2(gu.z); gf[4] = f.x; gf[5] = f.y; f = unpack_bf16x2(gu.w); gf[6] = f.x; gf[7] = f.y;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float gj = gf[j] * clip;
      mf[j] = a.beta1 * mf[j] + (1.0f - a.beta1) * gj;
      vf[j] = a.beta2 * vf[j] + (1.0f - a.beta2) * gj * gj;
      const float denom = sqrtf(vf[j]) / bc2s + a.eps;
      pf[j] = __fmul_rn(pf[j], decay) - step_size * mf[j] / denom;
    }
    reinterpret_cast<float4*>(a.p32)[2 * i] = make_float4(pf[0], pf[1], pf[2], pf[3]);
    reinterpret_cast<float4*>(a.p32)[2 * i + 1] = make_float4(pf[4], pf[5], pf[6], pf[7]);
    reinterpret_cast<uint4*>(a.p)[i] =
        make_uint4(pack_bf16x2(pf[0], pf[1]), pack_bf16x2(pf[2], pf[3]), pack_bf16x2(pf[4], pf[5]), pack_bf16x2(pf[6], pf[7]));
    reinterpret_cast<float4*>(a.m)[2 * i] = make_float4(mf[0], mf[1], mf[2], mf[3]);
    reinterpret_cast<float4*>(a.m)[2 * i + 1] = make_float4(mf[4], mf[5], mf[6], mf[7]);
    reinterpret_cast<float4*>(a.v)[2 * i] = make_float4(vf[0], vf[1], vf[2], vf[3]);
    reinterpret_cast<float4*>(a.v)[2 * i + 1] = make_float4(vf[4], vf[5], vf[6], vf[7]);
    if (a.zero_grad) reinterpret_cast<uint4*>(a.g)[i] = make_uint4(0, 0, 0, 0);
  }
  if (blockIdx.x == 0) {
    for (long long i = (nv << 3) + threadIdx.x; i < a.n; i += blockDim.x) {
      const float gj = __bfloat162float(a.g[i]) * clip;
      const float mj = a.beta1 * a.m[i] + (1.0f - a.beta1) * gj;
      const float vj = a.beta2 * a.v[i] + (1.0f - a.beta2) * gj * gj;
      a.m[i] = mj; a.v[i] = vj;
      const float denom = sqrtf(vj) / bc2s + a.eps;
      const float pj = __fmul_rn(a.p32[i], decay) - step_size * mj / denom;
      a.p32[i] = pj;
      a.p[i] = __float2bfloat16_rn(pj);
      if (a.zero_grad) a.g[i] = __float2bfloat16(0.f);
    }
  }
}
int adamw_master_dispatch(const dvla_adamw_master_args* a, cudaStream_t s) {
  if (!a || !a->p32 || !a->p || !a->g || !a->m || !a->v || !a->lr || !a->step) {
    set_error("adamw_master: null pointer");
    return DVLA_ERR_INVALID;
  }
  if ((reinterpret_cast<uintptr_t>(a->p32) | reinterpret_cast<uintptr_t>(a->p) | reinterpret_cast<uintptr_t>(a->g) |
       reinterpret_cast<uintptr_t>(a->m) | reinterpret_cast<uintptr_t>(a->v)) & 15) {
    set_error("adamw_master: buffers must be 16-byte aligned");
    return DVLA_ERR_INVALID;
  }
  if (a->n <= 0) return DVLA_OK;
  AdamWMasterParams k{a->p32, (bf16*)a->p, (bf16*)a->g, a->m, a->v, a->n, a->sumsq, a->lr, a->step,
                      a->beta1, a->beta2, a->eps, a->weight_decay, a->max_norm, a->grad_scale, a->zero_grad};
  adamw_master_kernel<<<grid_for(a->n, 256 * 8 * 2), 256, 0, s>>>(k);
  DVLA_CHECK_LAUNCH("adamw_master");
  return DVLA_OK;
}

}  // namespace dvla
