/* libdvla_sm90.so -- C ABI of the H100-native (sm_90a) DreamVLA hot path.
 *
 * The reference (Zhangwenyao1/DreamVLA @ 7145258) is 100 % Python and has no FFI of its own; every entry point
 * below replaces a PyTorch call site of the reference, cited as <file>:<line> into the reference tree.
 * The reference-side binding a maintainer would add is a ctypes stub (see INTEGRATION.md); the host-side mirror in
 * this repo is dreamvla_b200/_lib.py + dreamvla_b200/ops.py.
 *
 * Conventions
 *   - every function returns 0 on success, a negative dvla_status otherwise; dvla_last_error() gives the text
 *     (thread-local).  Nothing throws or aborts across the ABI.
 *   - all pointers are DEVICE pointers owned by the caller (PyTorch); kernels never allocate, free or synchronise,
 *     and launch only on the stream passed in (a cudaStream_t passed as void*).  All calls are CUDA-graph capturable.
 *   - bf16 tensors are raw uint16 storage; "ld*" are row strides in ELEMENTS.
 */
#ifndef DVLA_H_
#define DVLA_H_
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  DVLA_OK = 0,
  DVLA_ERR_INVALID = -1,     /* bad argument (shape / alignment / null) */
  DVLA_ERR_CUDA = -2,        /* CUDA runtime / driver error at launch */
  DVLA_ERR_UNSUPPORTED = -3  /* configuration outside what the kernels implement */
} dvla_status;

/* activation ids (epilogues of dvla_gemm, dvla_act_*) */
enum { DVLA_ACT_NONE = 0, DVLA_ACT_GELU_ERF = 1, DVLA_ACT_GELU_TANH = 2, DVLA_ACT_QUICK_GELU = 3, DVLA_ACT_RELU = 4,
       DVLA_ACT_SILU = 5 };

int dvla_version(void);
const char* dvla_last_error(void);
/* number of kernel launches issued by this library on the calling process since load (bench.py "gpu_launches") */
int64_t dvla_launch_count(void);

/* ---------------------------------------------------------------------------------------------------------------
 * GEMM + fused epilogue:   out[M,N] = epi( alpha * sum_k A(m,k) * B(n,k) )
 *   A(m,k) = a[m*lda + k]  (a_mn_major = 0, "K-major")   or a[k*lda + m]  (a_mn_major = 1)
 *   B(n,k) = b[n*ldb + k]  (b_mn_major = 0: nn.Linear weight [out,in])   or b[k*ldb + n] (1: HF Conv1D weight [in,out])
 *   epi(v): v += bias[n]; aux_out[m,n] = v (pre-activation, bf16);
 *           v = aux_in ? v * act'(aux_in[m,n]) : act(v);  v = dropout(v);  v += residual[m,n];  out[m,n] = v
 * Replaces: torch.nn.Linear / timm Mlp / timm Attention.qkv,proj (models/vit_mae.py:73-75, dreamvla_model.py:348-433,
 * action_model/models.py:130-134), HF Conv1D addmm (models/gpt2.py:53-54,292-293), the perceiver projections
 * (models/perceiver_resampler.py:14-17,31-33) and their autograd dgrad/wgrad.
 * Hot path: persistent warp-specialised wgmma (register accumulators, TMA-fed 128B-swizzled smem ring).
 * Operands whose strides/pointers are not 16-byte aligned run on a SIMT kernel of the same semantics.
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct {
  const void* a;         /* bf16 */
  const void* b;         /* bf16 */
  void* out;             /* bf16 (out_fp32 = 0) or fp32 (out_fp32 = 1) */
  const void* bias;      /* bf16 [N] or NULL */
  const void* residual;  /* same dtype as out, [M,N] stride ldr, or NULL; may alias out (accumulate) */
  void* aux_out;         /* bf16 [M,N] stride ld_aux or NULL */
  const void* aux_in;    /* bf16 [M,N] stride ld_aux or NULL (exclusive with aux_out) */
  int64_t M, N, K;
  int64_t lda, ldb, ldo, ldr, ld_aux;
  int32_t a_mn_major, b_mn_major;
  int32_t act;
  int32_t out_fp32;
  float alpha;
  float dropout_p;        /* in [0, 1), anything else (NaN too) is DVLA_ERR_INVALID; 0 disables */
  uint64_t dropout_seed;  /* RNG block = m*ceil(N/8) + n/8, bit n%8 (same convention as dvla_dropout) */
  const uint64_t* dropout_seed_ptr; /* optional DEVICE counter added to dropout_seed at run time (CUDA-graph replays) */
  /* optional scratch of >= dvla_gemm_workspace_bytes() bytes, 16-byte aligned, owned by one stream (calls on one stream may
   * share it).  Its first 64 KB are arrival counters: ZERO before the first call, left zero by every call; the rest holds
   * fp32 partial tiles and needs no initialisation.  With it, the output tiles that would form a partly filled last wave
   * are cut along K and summed in fp32 (fixed order) by the last unit to arrive.  It serves only that K-split tail: split-K
   * accumulations (out += A.B, the weight gradients) add each split's partial with bf16 red.global.add whether or not a
   * workspace is given.  NULL: no K-split tail. */
  void* workspace;
  int64_t workspace_bytes;
} dvla_gemm_args;
int dvla_gemm(const dvla_gemm_args* args, void* stream);

/* What dvla_gemm would launch for `args` (pointers are only tested for NULL and alignment, never dereferenced): host code only,
 * no CUDA call, so the tiling / split-K / K-split-tail decisions are testable without a GPU (tests/test_gemm_plan_cpu.py).
 * Work unit u of the persistent kernels covers k-blocks [kb0, kb1) of 64 of output tile `tile` (m fastest); tail_slot >= 0
 * marks a K-split tail unit (partial sums through the workspace), split its index among the tile's splits. */
typedef struct dvla_gemm_plan_info {
  int32_t kernel;                 /* 0 SIMT thread-per-8-outputs, 1 SIMT warp-per-8-outputs, 2 wgmma (3 is not used on sm_90) */
  int32_t tile_m, tile_n;         /* output tile of one CTA: 128 x 128 */
  int32_t m_tiles, n_tiles, k_blocks;
  int32_t k_splits, kb_per_split, atomic_out;     /* uniform split-K (weight gradients), bf16 red.global.add when atomic_out */
  int32_t tail_first, tail_splits, tail_kbps;     /* K-split tail: tiles >= tail_first are cut into tail_splits k-ranges */
  int32_t units, grid_ctas;
} dvla_gemm_plan_info;
int dvla_gemm_plan(const dvla_gemm_args* args, dvla_gemm_plan_info* out);
int dvla_gemm_plan_unit(const dvla_gemm_plan_info* plan, int32_t unit, int32_t* tile, int32_t* kb0, int32_t* kb1,
                        int32_t* tail_slot, int32_t* split);

/* ---------------------------------------------------------------------------------------------------------------
 * LayerNorm over the last dim (rows x D), optional affine.  fwd saves mean / rstd (fp32) for the backward.
 * Replaces nn.LayerNorm call sites: gpt2.py:326,333,477; timm Block norm1/norm2; perceiver_resampler.py:14,28-29,101;
 * dreamvla_model.py:279,352,...; DiT norms without affine (action_model/models.py:126,128,147).
 * bwd: dx, and dgamma/dbeta ACCUMULATED into fp32 workspaces [D] (caller zeroes, then dvla_cast adds into grads).
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct {
  const void* x;      /* bf16 [rows, D] stride ldx */
  const void* gamma;  /* bf16 [D] or NULL */
  const void* beta;   /* bf16 [D] or NULL */
  void* y;            /* bf16 [rows, D] stride ldy */
  float* mean;        /* fp32 [rows] or NULL (inference) */
  float* rstd;        /* fp32 [rows] or NULL */
  int64_t rows, D, ldx, ldy;
  float eps;
} dvla_layernorm_fwd_args;
int dvla_layernorm_fwd(const dvla_layernorm_fwd_args* args, void* stream);

typedef struct {
  const void* dy;     /* bf16 [rows, D] stride ld */
  const void* x;      /* bf16 [rows, D] stride ld */
  const void* gamma;  /* bf16 [D] or NULL */
  const float* mean;
  const float* rstd;
  void* dx;           /* bf16 [rows, D] stride ld ; may alias dy */
  float* dgamma;      /* fp32 [D] accumulated (atomicAdd) or NULL */
  float* dbeta;       /* fp32 [D] accumulated or NULL */
  int64_t rows, D, ld;
  const void* dres;   /* bf16 [rows, ld] or NULL: added to dx -- the gradient that reaches x through the residual branch that
                         forks off at the LayerNorm input (x + f(LN(x)) blocks), so no separate elementwise add is needed */
} dvla_layernorm_bwd_args;
int dvla_layernorm_bwd(const dvla_layernorm_bwd_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Multi-head attention, head_dim = 64 (96 on the short-sequence kernels), flash-style (no [Lq,Lk] score tensor in HBM).
 *   O[b,i,h,:] = softmax_j( scale * Q[b,i,h,:].K[b,j,h,:] + maskbias(i,j) ) V[b,j,h,:]
 * Q/K/V/O are addressed with element strides (batch, seq, head) so they can alias slices of a fused QKV buffer.
 * mask: NULL (all visible) or a bit matrix [Lq, mask_words] of uint32 (bit j%32 of word j/32 set = pair (i,j) visible),
 *       shared by all batches and heads -- the reference's additive {0,-inf} mask (dreamvla_model.py:25-66) as bits.
 * tile_flags: per (q-tile of 64, k-tile of 64) byte, 0 = skip, 1 = partial (consult bits), 2 = full; built by
 *       dvla_attn_mask_tiles from the bit matrix (NULL = all full).
 * lse: fp32 [B, H, Lq] log-sum-exp (natural log, of the scaled logits) saved for the backward, or NULL.
 * head_dim (last field, appended after version 100 shipped; 0 means 64, so zero-initialised structs keep their meaning):
 *       64 everywhere; 96 only where the short-sequence kernels run (Lq <= 32, Lk <= 64, no mask, no dropout; key_bias
 *       allowed) -- the DiT-S action head.  Anything else returns DVLA_ERR_UNSUPPORTED before any launch.
 * Replaces F.scaled_dot_product_attention (timm Attention; gpt2.py:266-273), eager _attn (gpt2.py:61-84) and the
 * einsum/softmax in PerceiverAttention (perceiver_resampler.py:55-59).
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct {
  const void* q; const void* k; const void* v;  /* bf16 */
  void* o;                                      /* bf16 */
  float* lse;
  const uint32_t* mask; const uint8_t* tile_flags;
  int64_t B, H, Lq, Lk;
  int64_t q_sb, q_ss, q_sh;   /* element strides: batch, sequence, head (head_dim contiguous) */
  int64_t k_sb, k_ss, k_sh;
  int64_t v_sb, v_ss, v_sh;
  int64_t o_sb, o_ss, o_sh;
  int32_t mask_words;         /* uint32 words per mask row */
  float scale;
  float dropout_p; uint64_t dropout_seed; /* attention-probability dropout (gpt2.py:272), p in [0, 1) (else DVLA_ERR_INVALID);
                                             RNG block = ((b*H+h)*Lq+i)*ceil(Lk/8)+j/8, bit j%8 */
  const uint64_t* dropout_seed_ptr;       /* optional device counter added to dropout_seed */
  const float* key_bias;      /* optional fp32 [Lk]: added to the scaled score of key j before the softmax (natural-log units).
                                 log(r) makes key j count r times -- the identical-mask-token form of a world decoder
                                 (dreamvla_model.py:803-806 with an all-zero position embedding).  Short-sequence kernels only
                                 (Lq <= 32, Lk <= 64, no mask, no dropout); DVLA_ERR_UNSUPPORTED otherwise. */
  int64_t head_dim;           /* 0 or 64, or 96 on the short-sequence kernels (see above) */
  /* Per-sequence masks (appended after version 100 shipped; NULL keeps the meaning above): `mask` and `tile_flags` are the
   * first of a stack of bit matrices / tile-flag arrays of one shape, and batch b attends under
   * mask + mask_index[b] * mask_stride with tile_flags + mask_index[b] * flags_stride.  mask_index is DEVICE int32 [B]; its
   * values must select matrices inside the caller's stack (not checked: the kernels read them).  Both mma.sync and wgmma
   * forward kernels honour it; a mask_index without a mask is DVLA_ERR_INVALID, as are negative strides. */
  const int32_t* mask_index;
  int64_t mask_stride;        /* uint32 words between consecutive bit matrices */
  int64_t flags_stride;       /* bytes between consecutive tile-flag arrays */
} dvla_attn_fwd_args;
int dvla_attn_fwd(const dvla_attn_fwd_args* args, void* stream);

typedef struct {
  const void* q; const void* k; const void* v; const void* o; const void* d_o; /* bf16 */
  const float* lse;
  float* delta;               /* fp32 workspace [B,H,Lq]: rowsum(dO*O) */
  void* dq; void* dk; void* dv; /* bf16, same strides as q/k/v */
  const uint32_t* mask; const uint8_t* tile_flags;
  int64_t B, H, Lq, Lk;
  int64_t q_sb, q_ss, q_sh, k_sb, k_ss, k_sh, v_sb, v_ss, v_sh, o_sb, o_ss, o_sh;
  int64_t do_sb, do_ss, do_sh;
  int64_t dq_sb, dq_ss, dq_sh, dk_sb, dk_ss, dk_sh, dv_sb, dv_ss, dv_sh;
  int32_t mask_words;
  float scale;
  float dropout_p; uint64_t dropout_seed;
  const uint64_t* dropout_seed_ptr;
  const uint32_t* mask_t;     /* optional TRANSPOSED bit matrix [Lk, mask_t_words] (bit i%32 of word i/32 of row j = pair (i,j)
                                 visible); accepted for ABI compatibility, not read by the sm_90 kernels */
  int32_t mask_t_words;
  const float* key_bias;      /* as in dvla_attn_fwd_args (a constant: receives no gradient) */
  int64_t head_dim;           /* as in dvla_attn_fwd_args */
} dvla_attn_bwd_args;
int dvla_attn_bwd(const dvla_attn_bwd_args* args, void* stream);

/* tile_flags[qt*num_kt + kt] from the bit mask; qt = ceil(Lq/64), kt = ceil(Lk/64). */
int dvla_attn_mask_tiles(const uint32_t* mask, int32_t mask_words, int64_t Lq, int64_t Lk, uint8_t* tile_flags,
                         void* stream);

/* The pretrain phase's per-forward observation-token drop (dreamvla_model.py:55-59), drawn on the device.
 * base_bits [L, mask_words]: the mask built with mask_l_obs_ratio = 0; layout: K timesteps of n_tok slots each (K*n_tok = L),
 * slots [num_A, num_A + n_obs) of a timestep are its observation tokens and the n_act slots after them its action tokens.
 * For timestep i and observation column j < n_obs the key is r(i, j) = philox4x32(seed + *seed_ptr, i*n_obs + j).x (word 0,
 * the 7-round Philox of the dropout masks; seed_ptr NULL counts as 0); the `count` columns with the smallest (r(i, j), j) are
 * dropped: bits (action rows of i) x (column i*n_tok + num_A + j) are cleared.  bits = base_bits otherwise (must not alias).
 * tile_flags [ceil(L/64), ceil(L/64)] is rebuilt from bits as by dvla_attn_mask_tiles.  No host reads, no allocation: the
 * call can be captured in a CUDA graph.  n_obs <= 256 and 0 <= count <= n_obs, else DVLA_ERR_INVALID. */
int dvla_attn_mask_obs_drop(const uint32_t* base_bits, uint32_t* bits, uint8_t* tile_flags, int32_t mask_words, int64_t L,
                            int64_t K, int64_t n_tok, int64_t num_A, int64_t n_obs, int64_t n_act, int64_t count,
                            uint64_t seed, const int64_t* seed_ptr, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Element-wise / reduction helpers
 * ------------------------------------------------------------------------------------------------------------- */
/* y[r, :] = sum over rows of x (column sum), accumulated into fp32 out[N]  (bias gradients). */
int dvla_colsum_accum(const void* x_bf16, int64_t rows, int64_t N, int64_t ld, float* out_fp32, void* stream);
/* dst_bf16[i] += (bf16) src_fp32[i]  (fold fp32 partial reductions into bf16 gradient buffers) */
int dvla_accum_fp32_into_bf16(const float* src, void* dst_bf16, int64_t n, void* stream);
/* y = dropout(x) with the same (seed, index) convention as the GEMM epilogue; in place allowed; used for
 * embd dropout (gpt2.py:459) and to re-apply an epilogue dropout mask to dY in the backward. */
int dvla_dropout(const void* x_bf16, void* y_bf16, int64_t rows, int64_t N, int64_t ldx, int64_t ldy, float p,
                 uint64_t seed, const uint64_t* seed_ptr, void* stream);
/* out[s, :a, :] = e[s]; out[s, a:, :] = m  -- rows shared by every sequence appended to per-sequence rows (the world
 * decoders' [query rows | mask-token rows] inputs, dreamvla_model.py:803-806).  e bf16 [n, a, C], m bf16 [b, C], out bf16
 * [n, a+b, C], all contiguous, C % 8 == 0. */
int dvla_cat_broadcast(const void* e_bf16, const void* m_bf16, void* out_bf16, int64_t n, int64_t a, int64_t b, int64_t C,
                       void* stream);
/* dx = dy * act'(pre)  */
int dvla_act_bwd(const void* dy_bf16, const void* pre_bf16, void* dx_bf16, int64_t n, int32_t act, void* stream);
/* The same, plus colsum_f32[c] += sum_r dx[r, c] in the same pass: the bias gradient of the layer whose pre-activation
 * `pre` is (what torch's AddmmBackward computes as grad.sum(0) after GeluBackward).  dy, pre, dx bf16 [rows, N]
 * contiguous; colsum fp32 [N], accumulated into (zero it for a plain sum). */
int dvla_act_bwd_colsum(const void* dy_bf16, const void* pre_bf16, void* dx_bf16, int64_t rows, int64_t N, int32_t act,
                        float* colsum_f32, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Fused losses: each writes  loss_out[0] += weight * loss  (fp32, device) and dpred = weight * dloss/dpred * gscale.
 * Replaces utils/train_utils.py:158-170,325-337,366-371,423-425,448-450,499-502 and utils/sigloss.py:11-15.
 * ------------------------------------------------------------------------------------------------------------- */
/* mean((pred*mask - label*mask)^2), mask per row (fp32 [rows] or NULL). */
int dvla_mse_loss(const void* pred_bf16, const void* label_bf16, const float* row_mask, int64_t rows, int64_t C,
                  float weight, float* loss_out, void* dpred_bf16, void* stream);
/* mean_rows(1 - cos(pred_row, label_row)) */
int dvla_cosine_loss(const void* pred_bf16, const void* label_bf16, int64_t rows, int64_t C, float weight,
                     float* loss_out, void* dpred_bf16, void* stream);
/* SiLog: two-phase; stats = fp32[2] workspace (sum d, sum d^2), zeroed by the caller. */
int dvla_silog_stats(const void* pred_bf16, const void* label_bf16, int64_t n, float* stats, void* stream);
int dvla_silog_finish(const void* pred_bf16, const void* label_bf16, int64_t n, const float* stats, float lambd,
                      float weight, float* loss_out, void* dpred_bf16, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Optimiser: global-norm clip + AdamW on flat buffers (utils/train_utils.py:600-608, train.py:174).
 *   dvla_sumsq: sumsq_out[0] += sum(g^2)            (fp32 accumulate; caller zeroes)
 *   dvla_adamw: clip = min(1, max_norm / (sqrt(sumsq) + 1e-6)); g *= clip * grad_scale; AdamW update of p (bf16) with
 *               fp32 moments; optionally zeroes g.  lr and step live on the device (no host sync per step).
 * ------------------------------------------------------------------------------------------------------------- */
int dvla_sumsq(const void* g_bf16, int64_t n, float* sumsq_out, void* stream);
typedef struct {
  void* p;            /* bf16 [n] */
  void* g;            /* bf16 [n] */
  float* m; float* v; /* fp32 [n] */
  int64_t n;
  const float* sumsq; /* fp32 [1] or NULL (no clipping) */
  const float* lr;    /* fp32 [1] device */
  const float* step;  /* fp32 [1] device: step count AFTER increment (>= 1) */
  float beta1, beta2, eps, weight_decay, max_norm, grad_scale;
  int32_t zero_grad;
} dvla_adamw_args;
int dvla_adamw(const dvla_adamw_args* args, void* stream);
/* dvla_adamw_master: the same clip + AdamW (same formula, same operation order) on fp32 MASTER weights p32, for
 * `--precision fp32`.  p32 is read and updated; the bf16 working copy p is written as round-to-nearest(p32) (exactly
 * p32.to(torch.bfloat16)) and never read.  Gradients stay bf16.  30 B of HBM traffic per parameter (dvla_adamw: 24).
 * All of p32, p, g, m, v 16-byte aligned. */
typedef struct {
  float* p32;         /* fp32 [n], read and written */
  void* p;            /* bf16 [n], written only */
  void* g;            /* bf16 [n] */
  float* m; float* v; /* fp32 [n] */
  int64_t n;
  const float* sumsq; /* fp32 [1] or NULL (gradient already clipped) */
  const float* lr;    /* fp32 [1] device */
  const float* step;  /* fp32 [1] device: step count AFTER increment (>= 1) */
  float beta1, beta2, eps, weight_decay, max_norm, grad_scale;
  int32_t zero_grad;
} dvla_adamw_master_args;
int dvla_adamw_master(const dvla_adamw_master_args* args, void* stream);
/* In-place clip of the accumulated gradient, every micro-step, as utils/train_utils.py:599-600 does
 * (clip_grad_norm_ on .grad that keeps accumulating):  g *= grad_scale * min(1, max_norm / (sqrt(sumsq)*grad_scale + 1e-6)). */
int dvla_grad_clip_scale(void* g_bf16, int64_t n, const float* sumsq, float max_norm, float grad_scale, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Fused action sampler: the DDIM loop of the DiT action head with classifier-free guidance as ONE persistent cooperative
 * kernel (replaces dreamvla_model.py:935-987 -> gaussian_diffusion.py:609-689 -> models.py:253-268 for one sequence).
 * batch must be 1 (rows = 2 guidance branches * 2T = 12); any other batch returns DVLA_ERR_UNSUPPORTED before any launch.
 * Every pointer is device memory, weights are bf16 nn.Linear layouts [out, in].
 * head_dim = hidden / heads must be 64 (DiT-B, DiT-L) or 96 (DiT-S); DVLA_ERR_UNSUPPORTED otherwise.
 * Schedule tables are HOST arrays of n_steps entries (respaced DDIM: timestep_map[i] is the original timestep of step i).
 * n_steps <= 12 (the prologue embeds every step's timestep as one row of a 12-row GEMM); DVLA_ERR_UNSUPPORTED otherwise.
 *
 * integrator (appended after version 100 shipped; 0 means DDIM, so zero-initialised structs keep their meaning):
 *   DVLA_DIT_DDIM     the eta = 0 DDIM update over timestep_map / the alpha tables, steps n_steps-1 .. 0; the start noise
 *                     is rounded to bf16 first (the module path casts it to the model dtype).
 *   DVLA_DIT_FM_EULER flow matching (`--use_fm`, FMDiffusion.ddim_sample_loop): steps 0 .. n_steps-1, the DiT's timestep
 *                     input of step i is t_values[i] (fp32, i / n_steps), the start state is the fp32 `noise` as given and
 *                     x += bf16((1 / n_steps) * u) with u the bf16 guided output.  timestep_map and the alpha tables are
 *                     not read (may be NULL); the module path forces cfg_scale to 1.0, callers that mirror it pass 1.0.
 *   Any other value returns DVLA_ERR_UNSUPPORTED, DVLA_DIT_FM_EULER with t_values NULL DVLA_ERR_INVALID, before any launch.
 * ------------------------------------------------------------------------------------------------------------- */
enum { DVLA_DIT_DDIM = 0, DVLA_DIT_FM_EULER = 1 };
typedef struct {
  const void *qkv_w, *qkv_b, *proj_w, *proj_b, *fc1_w, *fc1_b, *fc2_w, *fc2_b;   /* blocks.N.{attn.qkv, attn.proj, mlp.fc1, mlp.fc2} */
} dvla_dit_block_weights;
typedef struct {
  const dvla_dit_block_weights* blocks;  /* HOST array [depth] */
  int64_t depth, hidden, heads, mlp, token, freq, channels, T, batch;
  const void *x_w, *x_b;                 /* x_embedder.linear [hidden, channels], [hidden] */
  const void *t0_w, *t0_b, *t2_w, *t2_b; /* t_embedder.mlp.{0,2}: [hidden, freq], [hidden], [hidden, hidden], [hidden] */
  const void *z_w, *z_b, *uncondition;   /* z_embedder.linear [hidden, token], [hidden]; z_embedder.uncondition [token] */
  const void *pos;                       /* positional_embedding [2T, hidden] */
  const void *final_w, *final_b;         /* final_layer.linear [channels, hidden], [channels] */
  const void* z;                         /* bf16 [batch, T, token]: condition features (the backbone's action-token rows) */
  const float* noise;                    /* fp32 [batch, T, channels]: start state (DDIM noise, or the FM start state) */
  float* out;                            /* fp32 [batch, T, channels] */
  const int32_t* timestep_map;           /* HOST [n_steps] */
  const float *sqrt_recip_alphas_cumprod, *sqrt_recipm1_alphas_cumprod, *alphas_cumprod_prev;   /* HOST [n_steps] */
  int64_t n_steps;
  float cfg_scale;
  void* workspace; int64_t workspace_bytes;   /* >= dvla_dit_sampler_workspace_bytes(...) */
  int64_t integrator;                    /* DVLA_DIT_DDIM (0) or DVLA_DIT_FM_EULER (1), see above */
  const float* t_values;                 /* HOST [n_steps]: DiT timestep input of each step in execution order (FM only) */
} dvla_dit_sampler_args;
int64_t dvla_dit_sampler_workspace_bytes(int64_t batch, int64_t T, int64_t hidden, int64_t mlp, int64_t n_steps);
int dvla_dit_ddim_sample(const dvla_dit_sampler_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Device-side pieces of the reference's collator (utils/data_utils.py:1337-1354; SURVEY.md 8f-2).  dtype codes: 0 fp32, 1 bf16.
 *
 * dvla_shift_crop = RandomShiftsAug.forward / forward_traj (utils/data_utils.py:326-383) for GIVEN integer shifts:
 *   out[i, c, y, x] = x[i, c, clamp(y + sy_i - pad, 0, H-1), clamp(x + sx_i - pad, 0, W-1)],  shifts_xy int32 [n, 2] = (sx, sy)
 *   in [0, 2*pad] (the reference draws them with torch.randint(0 | 1, 2*pad+1) per image / per frame and feeds them to
 *   grid_sample on the replicate-padded image; every sample point is a pixel centre, so the op is this clamped crop).
 *   x, out: [n, c, H, W] contiguous; n = batch * frames for forward_traj.
 * dvla_resize_nearest = torchvision Resize((hout, wout), NEAREST) of depth_image_fn (utils/data_utils.py:3588-3603):
 *   out[i, y, x] = x[i, min(floor(y * hin/hout), hin-1), min(floor(x * win/wout), win-1)], scales in fp32 as torch computes them. */
int dvla_shift_crop(const void* x, void* out, const int32_t* shifts_xy, int64_t n, int64_t c, int64_t h, int64_t w, int32_t pad,
                    int32_t in_dtype, int32_t out_dtype, void* stream);
int dvla_resize_nearest(const float* x_f32, void* out, int64_t n, int64_t hin, int64_t win, int64_t hout, int64_t wout,
                        int32_t out_dtype, void* stream);

/* dvla_image_fn = CLIP's image transform `image_processor` (openai CLIP _transform(224): Resize(224, BICUBIC), CenterCrop(224),
 * ToTensor, Normalize) of 8-bit RGB frames, as the collator (utils/data_utils.py:175-179, :1311-1312) and the rollout wrappers
 * (utils/eval_utils_calvin.py:82-90, utils/eval_utils_libero.py:94-106) apply it through Pillow + torchvision, bit for bit:
 *   - resize: the short side becomes 224, the long side int(224 * long / short); a frame whose short side is 224 is not
 *     resampled.  Crop offsets int(round((size - 224) / 2)), Python's round (half to even).  Only the crop is computed.
 *   - Pillow's 8-bit resampling: horizontal pass, then vertical, each value clip8(2^21 + sum pixel * coeff) rounded to uint8
 *     between the passes; clip8(v) = 0 for v <= 0, 255 for v >= 2^30, v >> 22 otherwise.  Coefficient tables as
 *     dvla_bicubic_coeffs fills them: x* = (w, resized w, crop left, 224), y* = (h, resized h, crop top, 224).
 *   - out[i, ch, y, x] = lut[ch * 256 + v] for the resampled value v; the caller computes lut = (arange(256) / 255 - mean) / std
 *     (fp32 [3, 256]), so the output is ToTensor + Normalize's own arithmetic.
 * frames: uint8 [n, h, w, c] contiguous (HWC, what datasets and simulators hold), c must be 3, 1 <= h, w <= 3584 (a downscale
 * of at most 16x); out: [n, 3, 224, 224] fp32 / bf16 (out_dtype 0 / 1), 16-byte aligned.  flip_vertical != 0 reads the frame
 * bottom-up (LIBERO's agent view, utils/eval_utils_libero.py:96).  n = 0 is a no-op.  Bad arguments return DVLA_ERR_INVALID
 * without launching. */
typedef struct {
  const uint8_t* frames;
  void* out;
  int64_t n, h, w, c;
  const int32_t* xbounds; const int32_t* xcoeffs;     /* [224, 2], [224, dvla_bicubic_taps(w, resized w)] */
  const int32_t* ybounds; const int32_t* ycoeffs;     /* [224, 2], [224, dvla_bicubic_taps(h, resized h)] */
  const float* lut;                                   /* [3, 256] */
  int32_t flip_vertical;
  int32_t out_dtype;
} dvla_image_fn_args;
int dvla_image_fn(const dvla_image_fn_args* args, void* stream);

/* Pillow's bicubic resampling coefficients (Resample.c precompute_coeffs + normalize_coeffs_8bpc, a = -0.5, support
 * 2 * max(in/out, 1), double arithmetic, normalised by their sum, rounded half away from zero at 2^22) of a line of in_size
 * pixels resized to out_size, for the outputs [first, first + count).  Host code only, no CUDA call.
 *   bounds[2i] = first input pixel of output first + i, bounds[2i + 1] = its number of taps;
 *   coeffs[i * taps + k] = int32 coefficient of tap k, 0 past the used taps;  taps = dvla_bicubic_taps(in_size, out_size).
 * in_size == out_size is the identity (one tap of 2^22): Pillow skips a pass whose size does not change.
 * dvla_bicubic_taps returns the number of coefficients per output (Pillow's ksize), or a negative dvla_status. */
int32_t dvla_bicubic_taps(int64_t in_size, int64_t out_size);
int dvla_bicubic_coeffs(int64_t in_size, int64_t out_size, int64_t first, int64_t count, int32_t* bounds, int32_t* coeffs);

/* SM budget of the persistent GEMM and attention-backward kernels (one CTA / CTA pair per SM).  0 = all SMs (default).
 * The data-parallel train step lowers it by the number of CTAs the NCCL all-reduce occupies while gradient exchange
 * overlaps the backward pass (train.py:173 DDP overlap), so that every persistent CTA is resident at once.  Returns the
 * previous value.  Process-wide. */
int dvla_set_sm_budget(int n_sms);

/* ---------------------------------------------------------------------------------------------------------------
 * Workspace sizes (bytes) of the ops that need caller-provided scratch -- the library never allocates device memory:
 *   attn_bwd : `delta` fp32 [B, H, Lq]  (rowsum(dO * O), FlashAttention-2 backward)
 *   silog    : `stats` fp32 [2]         (sum d, sum d^2; zeroed by the caller before dvla_silog_stats)
 *   gemm     : optional (dvla_gemm_args.workspace): fp32 partial tiles + arrival counters of the K-split tail
 * ------------------------------------------------------------------------------------------------------------- */
int64_t dvla_attn_bwd_workspace_bytes(int64_t B, int64_t H, int64_t Lq);
int64_t dvla_silog_workspace_bytes(void);
int64_t dvla_gemm_workspace_bytes(const dvla_gemm_args* args);

#ifdef __cplusplus
}
#endif
#endif /* DVLA_H_ */
