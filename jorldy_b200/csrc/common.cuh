// Shared device/host helpers for the jorldy_b200 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define JB_OK 0
#define JB_ERR_INVALID (-22)   /* EINVAL-style: bad argument */
#define JB_ERR_CUDA (-5)       /* EIO-style: CUDA launch / runtime failure */

#define JB_SM_COUNT 132        /* H100 SXM */

#define JB_API extern "C" __attribute__((visibility("default")))

static inline int jb_check_launch() {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? JB_OK : JB_ERR_CUDA;
}

static inline int jb_div_up(long long a, long long b) { return (int)((a + b - 1) / b); }

// Persistent-style grid size: enough CTAs to cover `work` items at `per_cta`
// items each, rounded up to whole waves of the 132 SMs, capped at `max_waves`.
static inline int jb_grid_for(long long work, int per_cta, int max_waves = 32) {
  long long ctas = (work + per_cta - 1) / per_cta;
  if (ctas < 1) ctas = 1;
  long long cap = (long long)JB_SM_COUNT * max_waves;
  if (ctas > cap) ctas = cap;
  return (int)ctas;
}

__device__ __forceinline__ float jb_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double jb_warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float jb_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float jb_warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
