// Host-side plumbing shared by the .cu files of libdvla_sm90.so: error text, launch accounting, the SM budget and launch
// grids, the alignment test, the tensor-map encoder and the dropout-rate policy.  Host code only.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <mutex>

#include "../../include/dvla.h"

namespace dvla {

// state.cu
void set_error(const char* fmt, ...);   // sets the thread's dvla_last_error() text
void count_launch();
int num_sms();

// After a kernel launch: a launch error sets "<name> launch: <CUDA error>" and returns DVLA_ERR_CUDA from the caller; a
// successful launch is counted in dvla_launch_count().
#define DVLA_CHECK_LAUNCH(name)                                                                                 \
  do {                                                                                                          \
    cudaError_t e__ = cudaGetLastError();                                                                       \
    if (e__ != cudaSuccess) { set_error("%s launch: %s", name, cudaGetErrorString(e__)); return DVLA_ERR_CUDA; } \
    count_launch();                                                                                             \
  } while (0)

// cuTensorMapEncodeTiled through the runtime's driver entry point (gemm_sm90.cu); NULL if the driver lacks it.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode_fn();

// cudaFuncSetAttribute once per kernel instantiation (the caller's static `once` and `err`), race-free between the
// forward and the autograd thread; false if it failed, with the error in `err`.
template <typename K>
bool set_smem_attr_once(std::once_flag& once, cudaError_t& err, K kern, int bytes) {
  std::call_once(once, [&] { err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes); });
  return err == cudaSuccess;
}

// Blocks for a grid-stride loop over work_items at per_block items per block: ceil(work_items / per_block), clamped to
// [1, blocks_per_sm * SMs].
inline unsigned grid_for(long long work_items, long long per_block, int blocks_per_sm) {
  long long b = (work_items + per_block - 1) / per_block;
  const long long cap = (long long)blocks_per_sm * num_sms();
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (unsigned)b;
}

// Grid of a column-sum kernel over [rows, N]: x = one block per 256-column slab, y = row chunks of *rows_per_block rows,
// about blocks_per_sm blocks per SM in all, and no chunk under min_rows_per_block rows unless rows is smaller.
inline dim3 slab_grid(long long rows, long long N, int blocks_per_sm, int min_rows_per_block, int* rows_per_block) {
  const int bx = (int)((N + 255) / 256);
  long long by = ((long long)blocks_per_sm * num_sms() + bx - 1) / bx;
  if (by > (rows + min_rows_per_block - 1) / min_rows_per_block) by = (rows + min_rows_per_block - 1) / min_rows_per_block;
  if (by < 1) by = 1;
  *rows_per_block = (int)((rows + by - 1) / by);
  return dim3(bx, (unsigned)((rows + *rows_per_block - 1) / *rows_per_block));
}

// True if every pointer is 16-byte aligned, as the kernels' 16-byte vector accesses need.
template <class... T>
inline bool aligned16(const T*... p) {
  return ((reinterpret_cast<uintptr_t>(p) | ... | uintptr_t(0)) & 15) == 0;
}

// Dropout rates the ABI accepts: [0, 1).  Written so that NaN fails too.
inline bool dropout_rate_ok(float p) { return p >= 0.f && p < 1.f; }

// A rate as the kernels apply it: an element is dropped when its 16-bit draw is below thresh = round(p * 65536), and the
// kept ones are scaled by 1 / (1 - thresh / 65536).  tests/philox_ref.py restates both roundings.
inline void dropout_thresh_scale(float p, uint32_t* thresh, float* scale) {
  *thresh = (uint32_t)(p * 65536.0f + 0.5f);
  *scale = 1.0f / (1.0f - (float)*thresh / 65536.0f);
}

}  // namespace dvla
