// Host-side plumbing shared by the .cu files of libdvla_sm90.so: error text, launch accounting, the SM budget, the
// tensor-map encoder and the dropout-rate policy.  Host code only.
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

// Dropout rates the ABI accepts: [0, 1).  Written so that NaN fails too.
inline bool dropout_rate_ok(float p) { return p >= 0.f && p < 1.f; }

// A rate as the kernels apply it: an element is dropped when its 16-bit draw is below thresh = round(p * 65536), and the
// kept ones are scaled by 1 / (1 - thresh / 65536).  tests/philox_ref.py restates both roundings.
inline void dropout_thresh_scale(float p, uint32_t* thresh, float* scale) {
  *thresh = (uint32_t)(p * 65536.0f + 0.5f);
  *scale = 1.0f / (1.0f - (float)*thresh / 65536.0f);
}

}  // namespace dvla
