// extern "C" entry points of libdvla_sm90.so (declared in include/dvla.h): argument validation, error text,
// launch accounting.  No torch types cross this boundary.
#include <atomic>
#include <stdarg.h>
#include <stdio.h>

#include "../../include/dvla.h"
#include "common.cuh"

namespace dvla {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
static std::atomic<int> g_sm_budget{0};
// SMs the persistent kernels (one CTA, or CTA pair, per SM) may size their grids for: the device's SM count, or the
// caller's budget while a collective shares the GPU (dvla_set_sm_budget) -- a persistent grid that cannot place every CTA
// runs its stragglers as a second wave.
int num_sms() {
  static const int n = [] {
    int dev = 0, v = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;   // H100 SXM
    return v;
  }();
  const int b = g_sm_budget.load(std::memory_order_relaxed);
  return (b > 0 && b < n) ? b : n;
}

int gemm_dispatch(const dvla_gemm_args* a, cudaStream_t stream);
int64_t gemm_workspace_bytes();
int shift_crop_dispatch(const void* x, void* out, const int32_t* shifts, int64_t n, int64_t c, int64_t h, int64_t w, int32_t pad,
                        int32_t in_dtype, int32_t out_dtype, cudaStream_t s);
int resize_nearest_dispatch(const float* x, void* out, int64_t n, int64_t hin, int64_t win, int64_t hout, int64_t wout,
                            int32_t out_dtype, cudaStream_t s);
int gemm_plan(const dvla_gemm_args* a, dvla_gemm_plan_info* out);
int gemm_plan_unit(const dvla_gemm_plan_info* plan, int unit, int* tile, int* kb0, int* kb1, int* slot, int* split);
int layernorm_fwd_dispatch(const dvla_layernorm_fwd_args* a, cudaStream_t stream);
int layernorm_bwd_dispatch(const dvla_layernorm_bwd_args* a, cudaStream_t stream);
int attn_fwd_dispatch(const dvla_attn_fwd_args* a, cudaStream_t stream);
int attn_bwd_dispatch(const dvla_attn_bwd_args* a, cudaStream_t stream);
int attn_mask_tiles_dispatch(const uint32_t* mask, int32_t mask_words, int64_t Lq, int64_t Lk, uint8_t* flags,
                             cudaStream_t stream);
int colsum_accum_dispatch(const void* x, int64_t rows, int64_t N, int64_t ld, float* out, cudaStream_t s);
int accum_fp32_into_bf16_dispatch(const float* src, void* dst, int64_t n, cudaStream_t s);
int dropout_dispatch(const void* x, void* y, int64_t rows, int64_t N, int64_t ldx, int64_t ldy, float p, uint64_t seed,
                     const uint64_t* seed_ptr, cudaStream_t s);
int cat_broadcast_dispatch(const void* e, const void* m, void* out, int64_t n, int64_t a, int64_t b, int64_t C, cudaStream_t s);
int dit_ddim_sample_dispatch(const dvla_dit_sampler_args* a, cudaStream_t s);
int act_bwd_dispatch(const void* dy, const void* pre, void* dx, int64_t n, int32_t act, cudaStream_t s);
int act_bwd_colsum_dispatch(const void* dy, const void* pre, void* dx, int64_t rows, int64_t N, int32_t act, float* colsum,
                            cudaStream_t s);
int mse_loss_dispatch(const void* pred, const void* label, const float* row_mask, int64_t rows, int64_t C, float weight,
                      float* loss_out, void* dpred, cudaStream_t s);
int cosine_loss_dispatch(const void* pred, const void* label, int64_t rows, int64_t C, float weight, float* loss_out,
                         void* dpred, cudaStream_t s);
int silog_stats_dispatch(const void* pred, const void* label, int64_t n, float* stats, cudaStream_t s);
int silog_finish_dispatch(const void* pred, const void* label, int64_t n, const float* stats, float lambd, float weight,
                          float* loss_out, void* dpred, cudaStream_t s);
int sumsq_dispatch(const void* g, int64_t n, float* out, cudaStream_t s);
int adamw_dispatch(const dvla_adamw_args* a, cudaStream_t s);
int adamw_master_dispatch(const dvla_adamw_master_args* a, cudaStream_t s);
int grad_clip_scale_dispatch(void* g, int64_t n, const float* sumsq, float max_norm, float grad_scale, cudaStream_t s);

}  // namespace dvla

using namespace dvla;
#define S(stream) reinterpret_cast<cudaStream_t>(stream)

extern "C" {

int dvla_version(void) { return 100; }
const char* dvla_last_error(void) { return g_err; }
int64_t dvla_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int dvla_gemm(const dvla_gemm_args* args, void* stream) { return gemm_dispatch(args, S(stream)); }
int dvla_gemm_plan(const dvla_gemm_args* args, dvla_gemm_plan_info* out) { return gemm_plan(args, out); }
int dvla_gemm_plan_unit(const dvla_gemm_plan_info* plan, int32_t unit, int32_t* tile, int32_t* kb0, int32_t* kb1,
                        int32_t* tail_slot, int32_t* split) {
  return gemm_plan_unit(plan, unit, tile, kb0, kb1, tail_slot, split);
}
int dvla_layernorm_fwd(const dvla_layernorm_fwd_args* a, void* stream) { return layernorm_fwd_dispatch(a, S(stream)); }
int dvla_layernorm_bwd(const dvla_layernorm_bwd_args* a, void* stream) { return layernorm_bwd_dispatch(a, S(stream)); }
int dvla_attn_fwd(const dvla_attn_fwd_args* a, void* stream) { return attn_fwd_dispatch(a, S(stream)); }
int dvla_attn_bwd(const dvla_attn_bwd_args* a, void* stream) { return attn_bwd_dispatch(a, S(stream)); }
int dvla_attn_mask_tiles(const uint32_t* mask, int32_t mask_words, int64_t Lq, int64_t Lk, uint8_t* tile_flags,
                         void* stream) {
  return attn_mask_tiles_dispatch(mask, mask_words, Lq, Lk, tile_flags, S(stream));
}
int dvla_colsum_accum(const void* x, int64_t rows, int64_t N, int64_t ld, float* out, void* stream) {
  return colsum_accum_dispatch(x, rows, N, ld, out, S(stream));
}
int dvla_accum_fp32_into_bf16(const float* src, void* dst, int64_t n, void* stream) {
  return accum_fp32_into_bf16_dispatch(src, dst, n, S(stream));
}
int dvla_dropout(const void* x, void* y, int64_t rows, int64_t N, int64_t ldx, int64_t ldy, float p, uint64_t seed,
                 const uint64_t* seed_ptr, void* stream) {
  return dropout_dispatch(x, y, rows, N, ldx, ldy, p, seed, seed_ptr, S(stream));
}
int dvla_cat_broadcast(const void* e, const void* m, void* out, int64_t n, int64_t a, int64_t b, int64_t C, void* stream) {
  return cat_broadcast_dispatch(e, m, out, n, a, b, C, S(stream));
}
int dvla_act_bwd(const void* dy, const void* pre, void* dx, int64_t n, int32_t act, void* stream) {
  return act_bwd_dispatch(dy, pre, dx, n, act, S(stream));
}
int dvla_shift_crop(const void* x, void* out, const int32_t* shifts_xy, int64_t n, int64_t c, int64_t h, int64_t w, int32_t pad,
                    int32_t in_dtype, int32_t out_dtype, void* stream) {
  return shift_crop_dispatch(x, out, shifts_xy, n, c, h, w, pad, in_dtype, out_dtype, S(stream));
}
int dvla_resize_nearest(const float* x, void* out, int64_t n, int64_t hin, int64_t win, int64_t hout, int64_t wout,
                        int32_t out_dtype, void* stream) {
  return resize_nearest_dispatch(x, out, n, hin, win, hout, wout, out_dtype, S(stream));
}
int dvla_act_bwd_colsum(const void* dy, const void* pre, void* dx, int64_t rows, int64_t N, int32_t act, float* colsum,
                        void* stream) {
  return act_bwd_colsum_dispatch(dy, pre, dx, rows, N, act, colsum, S(stream));
}
int dvla_mse_loss(const void* pred, const void* label, const float* row_mask, int64_t rows, int64_t C, float weight,
                  float* loss_out, void* dpred, void* stream) {
  return mse_loss_dispatch(pred, label, row_mask, rows, C, weight, loss_out, dpred, S(stream));
}
int dvla_cosine_loss(const void* pred, const void* label, int64_t rows, int64_t C, float weight, float* loss_out,
                     void* dpred, void* stream) {
  return cosine_loss_dispatch(pred, label, rows, C, weight, loss_out, dpred, S(stream));
}
int dvla_silog_stats(const void* pred, const void* label, int64_t n, float* stats, void* stream) {
  return silog_stats_dispatch(pred, label, n, stats, S(stream));
}
int dvla_silog_finish(const void* pred, const void* label, int64_t n, const float* stats, float lambd, float weight,
                      float* loss_out, void* dpred, void* stream) {
  return silog_finish_dispatch(pred, label, n, stats, lambd, weight, loss_out, dpred, S(stream));
}
int dvla_sumsq(const void* g, int64_t n, float* out, void* stream) { return sumsq_dispatch(g, n, out, S(stream)); }
int dvla_adamw(const dvla_adamw_args* a, void* stream) { return adamw_dispatch(a, S(stream)); }
int dvla_adamw_master(const dvla_adamw_master_args* a, void* stream) { return adamw_master_dispatch(a, S(stream)); }
int dvla_grad_clip_scale(void* g, int64_t n, const float* sumsq, float max_norm, float grad_scale, void* stream) {
  return grad_clip_scale_dispatch(g, n, sumsq, max_norm, grad_scale, S(stream));
}

int dvla_dit_ddim_sample(const dvla_dit_sampler_args* a, void* stream) { return dit_ddim_sample_dispatch(a, S(stream)); }
int dvla_set_sm_budget(int n_sms) {
  const int prev = g_sm_budget.exchange(n_sms > 0 ? (n_sms & ~1) : 0, std::memory_order_relaxed);   // even: CTA pairs
  return prev;
}
int64_t dvla_attn_bwd_workspace_bytes(int64_t B, int64_t H, int64_t Lq) { return (B > 0 && H > 0 && Lq > 0) ? 4 * B * H * Lq : 0; }
int64_t dvla_silog_workspace_bytes(void) { return 2 * (int64_t)sizeof(float); }
int64_t dvla_gemm_workspace_bytes(const dvla_gemm_args* args) { (void)args; return gemm_workspace_bytes(); }

}  // extern "C"
