// Shared device helpers for the sm_90a kernels: mbarrier, TMA, wgmma PTX wrappers,
// bf16 packing, warp reductions and a counter-based RNG for dropout.
// Everything here is hand-written inline PTX for sm_90a (no CUTLASS dependency in the build).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace dvla {

typedef __nv_bfloat16 bf16;

#ifndef DVLA_WATCHDOG_CYCLES
#define DVLA_WATCHDOG_CYCLES (4000000000ll)  // ~2 s at 2 GHz: turn a protocol hang into a trap
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// kReport = false: the same watchdog without the diagnostic printf.  printf is a function call, and a call anywhere in a
// function that issues wgmma makes ptxas serialise every wgmma of that function.
template <bool kReport = true>
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  uint32_t spins = 0;
  long long t0 = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3FFu) == 0) {                  // watchdog: look at the clock only every 1024 failed polls
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > DVLA_WATCHDOG_CYCLES) {
        if (kReport) printf("dvla: mbarrier watchdog (block %d thread %d parity %u)\n", blockIdx.x, threadIdx.x, parity);
        __trap();
      }
    }
  }
}

// Hand registers between warpgroups of a warp-specialised kernel (per-warpgroup register budget, sm_90a).
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// ---------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor), 2-D and 3-D tiled loads into shared memory, completion on mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], "
      "[%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// ---------------------------------------------------------------------------------------------
// wgmma (sm_90a warpgroup MMA): D[64 x 128] fp32 in registers (+)= A[smem desc] * B[smem desc], bf16 inputs.
// Issued by all 128 threads of a warpgroup.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Keeps the compiler from moving reads or writes of the accumulator across a wgmma_wait.
__device__ __forceinline__ void wgmma_fence_operand(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Accumulator layout (per warp w of the warpgroup, lane l): d[4*j + 2*h + e] is row 16*w + l/4 + 8*h, column
// 8*j + 2*(l%4) + e.  TA / TB = 1 reads that operand MN-major (transposed) from shared memory.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16_bf16(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(TA), "n"(TB)
      : "memory");
}

// D[64 x 64] fp32 (+)= A[smem desc] * B[smem desc]; both operands K-major.
__device__ __forceinline__ void wgmma_m64n64k16_ss(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
// D[64 x 64] fp32 += A[registers] * B[smem desc, MN-major]; A is the bf16 fragment of mma.sync m16n8k16 for this warp's 16
// rows (a[0..3]), so an accumulator of this shape converts to the next A operand without leaving registers.
__device__ __forceinline__ void wgmma_m64n64k16_rs_tb(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, 1, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b)
      : "memory");
}
__device__ __forceinline__ void wgmma_fence_operand32(float (&d)[32]) {
#pragma unroll
  for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// wgmma shared-memory matrix descriptor (sm_90), 128-byte swizzle.
//   bits [0,14) start address >> 4    bits [16,30) leading byte offset >> 4    bits [32,46) stride byte offset >> 4
//   bits [62,64) layout type (1 = SWIZZLE_128B).  Tiles are 1024-byte aligned, so the base-offset field stays 0.
// K-major tile  (rows x 64 bf16, one 128 B swizzle row per matrix row): SBO = 1024 (8 rows), LBO unused.
// MN-major tile (64-wide MN atoms, K rows of 128 B): SBO = 1024 (8 K-rows), LBO = bytes between 64-wide MN atoms.
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// Named barrier over `count` threads (ids 1.. ; 0 is __syncthreads).
__device__ __forceinline__ void named_barrier_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ---------------------------------------------------------------------------------------------
// misc math
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
// One 16-byte vector of 8 bf16 <-> 8 fp32.  The caller issues the load or store (plain, __ldg, ld.cg, ...).
__device__ __forceinline__ void unpack_bf16x8(const uint4& u, float (&f)[8]) {
  float2 t;
  t = unpack_bf16x2(u.x); f[0] = t.x; f[1] = t.y;
  t = unpack_bf16x2(u.y); f[2] = t.x; f[3] = t.y;
  t = unpack_bf16x2(u.z); f[4] = t.x; f[5] = t.y;
  t = unpack_bf16x2(u.w); f[6] = t.x; f[7] = t.y;
}
__device__ __forceinline__ uint4 pack_bf16x8(const float (&f)[8]) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}
// The same with a plain 16-byte load / store at p (16-byte aligned).  The load goes to a local first: a reference bound to
// the memory itself would let the compiler split it into four 4-byte loads.
__device__ __forceinline__ void load_bf16x8(const bf16* p, float (&f)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  unpack_bf16x8(u, f);
}
__device__ __forceinline__ void store_bf16x8(bf16* p, const float (&f)[8]) { *reinterpret_cast<uint4*>(p) = pack_bf16x8(f); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Activations (fp32 math).  Ids are part of the C ABI (include/dvla.h).
enum Act : int { ACT_NONE = 0, ACT_GELU_ERF = 1, ACT_GELU_TANH = 2, ACT_QUICK_GELU = 3, ACT_RELU = 4, ACT_SILU = 5 };

// Branch-free approximate reciprocal / exp2 (single MUFU each).  The IEEE variants (`/`, __frcp_rn, expf) compile to a MUFU
// plus a guarded slow path -- one branch per element -- which makes an epilogue of a few flops per element instruction-bound.
__device__ __forceinline__ float rcp_approx(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float sigmoid_fast(float x) {   // 1 / (1 + e^-x)
  return rcp_approx(1.0f + ex2_approx(-1.4426950408889634f * x));
}
// erf with |abs error| <= 1.5e-7 + MUFU approximation error (Abramowitz & Stegun 7.1.26): ~16 branch-free instructions.
__device__ __forceinline__ float fast_erf(float x) {
  const float ax = fabsf(x);
  const float t = rcp_approx(fmaf(0.3275911f, ax, 1.0f));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float e = ex2_approx(ax * ax * -1.4426950408889634f);
  const float r = fmaf(-p * t, e, 1.0f);
  return copysignf(r, x);
}

__device__ __forceinline__ float act_fwd(float x, int act) {
  switch (act) {
    case ACT_GELU_ERF: {
      const float hx = 0.5f * x;
      return fmaf(hx, fast_erf(x * 0.70710678118654752f), hx);
    }
    case ACT_GELU_TANH: {  // 0.5x(1+tanh(u)) == x*sigmoid(2u)
      const float u = x * fmaf(0.0356774081f, x * x, 0.7978845608028654f);   // sqrt(2/pi)(x + 0.044715x^3)
      return x * sigmoid_fast(2.0f * u);
    }
    case ACT_QUICK_GELU: return x * sigmoid_fast(1.702f * x);
    case ACT_RELU: return fmaxf(x, 0.0f);
    case ACT_SILU: return x * sigmoid_fast(x);
    default: return x;
  }
}
// Apply an activation to n values with the switch hoisted out of the element loop.
template <int N>
__device__ __forceinline__ void act_fwd_n(float (&v)[N], int act) {
  switch (act) {
    case ACT_GELU_ERF:
#pragma unroll
      for (int j = 0; j < N; ++j) v[j] = act_fwd(v[j], ACT_GELU_ERF);
      break;
    case ACT_GELU_TANH:
#pragma unroll
      for (int j = 0; j < N; ++j) v[j] = act_fwd(v[j], ACT_GELU_TANH);
      break;
    case ACT_QUICK_GELU:
#pragma unroll
      for (int j = 0; j < N; ++j) v[j] = act_fwd(v[j], ACT_QUICK_GELU);
      break;
    case ACT_RELU:
#pragma unroll
      for (int j = 0; j < N; ++j) v[j] = fmaxf(v[j], 0.f);
      break;
    case ACT_SILU:
#pragma unroll
      for (int j = 0; j < N; ++j) v[j] = act_fwd(v[j], ACT_SILU);
      break;
    default: break;
  }
}

// d act(x) / dx evaluated at the pre-activation x.
__device__ __forceinline__ float act_bwd(float x, int act) {
  switch (act) {
    case ACT_GELU_ERF: {
      const float cdf = fmaf(0.5f, fast_erf(x * 0.70710678118654752f), 0.5f);
      const float pdf = 0.3989422804014327f * ex2_approx(x * x * -0.7213475204444817f);   // exp(-x^2/2)/sqrt(2pi)
      return fmaf(x, pdf, cdf);
    }
    case ACT_GELU_TANH: {
      const float x2 = x * x;
      const float u = x * fmaf(0.0356774081f, x2, 0.7978845608028654f);
      const float s = sigmoid_fast(2.0f * u);
      const float du = fmaf(0.1070322243f, x2, 0.7978845608028654f);            // sqrt(2/pi)(1 + 3*0.044715 x^2)
      return fmaf(x * s * (1.0f - s), 2.0f * du, s);
    }
    case ACT_QUICK_GELU: {
      const float s = sigmoid_fast(1.702f * x);
      return fmaf(1.702f * x * s, 1.0f - s, s);
    }
    case ACT_RELU: return x > 0.0f ? 1.0f : 0.0f;
    case ACT_SILU: {
      const float s = sigmoid_fast(x);
      return fmaf(x * s, 1.0f - s, s);
    }
    default: return 1.0f;
  }
}

// v[j] *= act'(x[j]) with the switch hoisted out of the element loop.
template <int N>
__device__ __forceinline__ void act_bwd_mul_n(float (&v)[N], const float (&x)[N], int act) {
  switch (act) {
    case ACT_GELU_ERF:
#pragma unroll
      for (int j = 0; j < N; ++j) v[j] *= act_bwd(x[j], ACT_GELU_ERF);
      break;
    case ACT_GELU_TANH:
#pragma unroll
      for (int j = 0; j < N; ++j) v[j] *= act_bwd(x[j], ACT_GELU_TANH);
      break;
    case ACT_QUICK_GELU:
#pragma unroll
      for (int j = 0; j < N; ++j) v[j] *= act_bwd(x[j], ACT_QUICK_GELU);
      break;
    case ACT_RELU:
#pragma unroll
      for (int j = 0; j < N; ++j) v[j] = x[j] > 0.f ? v[j] : 0.f;
      break;
    case ACT_SILU:
#pragma unroll
      for (int j = 0; j < N; ++j) v[j] *= act_bwd(x[j], ACT_SILU);
      break;
    default: break;
  }
}

// Counter-based RNG (Philox-4x32, Salmon et al. SC'11).  One call yields 4 uniform 32-bit words for (seed, offset).
// 7 rounds: the smallest round count the authors report as passing BigCrush (curand's default of 10 adds margin only);
// the dropout masks need independent Bernoulli draws, not cryptographic strength, and the RNG dominates the instructions of
// the attention kernels' dropout path.
constexpr int DVLA_PHILOX_ROUNDS = 7;
__device__ __forceinline__ uint4 philox4x32(uint64_t seed, uint64_t offset) {
  uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
  uint32_t c0 = static_cast<uint32_t>(offset), c1 = static_cast<uint32_t>(offset >> 32), c2 = 0x243F6A88u, c3 = 0x85A308D3u;
#pragma unroll
  for (int i = 0; i < DVLA_PHILOX_ROUNDS; ++i) {
    uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}
// Dropout keep-mask for the 8 consecutive elements [8*blk, 8*blk+8): 16 random bits per element,
// element j of the block is kept iff its 16-bit draw >= thresh (thresh = round(p * 65536)).
// Returned as an 8-bit mask.  Forward and backward regenerate the same mask from (seed, element index).
__device__ __forceinline__ uint32_t dropout_keep8(uint64_t seed, uint64_t blk, uint32_t thresh) {
  uint4 r = philox4x32(seed, blk);
  uint32_t m = 0;
  m |= ((r.x & 0xFFFFu) >= thresh) << 0; m |= ((r.x >> 16) >= thresh) << 1;
  m |= ((r.y & 0xFFFFu) >= thresh) << 2; m |= ((r.y >> 16) >= thresh) << 3;
  m |= ((r.z & 0xFFFFu) >= thresh) << 4; m |= ((r.z >> 16) >= thresh) << 5;
  m |= ((r.w & 0xFFFFu) >= thresh) << 6; m |= ((r.w >> 16) >= thresh) << 7;
  return m;
}
// The same mask without materialising it: element j of the block whose Philox words are `r` is kept iff its 16-bit draw
// (low half of word j/2 for even j, high half for odd j) >= thresh.  `th16` = thresh << 16, so the high half compares as
// the whole word and the low half after one shift: 1-2 instructions per element instead of ~6 to build and test mask bits.
__device__ __forceinline__ bool dropout_keep_elem(const uint4& r, uint32_t th16, int j) {
  const uint32_t w = j < 2 ? r.x : j < 4 ? r.y : j < 6 ? r.z : r.w;
  return (j & 1) ? (w >= th16) : ((w << 16) >= th16);
}

}  // namespace dvla
