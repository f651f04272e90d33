// common.cuh -- shared helpers for the nerf_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "../../include/nerf_b200.h"

namespace nb {

// ---- error reporting -------------------------------------------------------------------------
extern thread_local char g_err[512];
extern long long g_launches;
int set_error(int code, const char* fmt, ...);

#define NB_CHECK_ARG(cond, ...) do { if (!(cond)) return nb::set_error(-2, __VA_ARGS__); } while (0)
#define NB_CUDA(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) \
    return nb::set_error(-3, "%s failed: %s", #expr, cudaGetErrorString(e__)); } while (0)
#define NB_LAUNCH_OK(name) do { nb::g_launches++; cudaError_t e__ = cudaPeekAtLastError(); \
    if (e__ != cudaSuccess) { (void)cudaGetLastError(); \
      return nb::set_error(-4, "launch of %s failed: %s", name, cudaGetErrorString(e__)); } } while (0)

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// ---- warp helpers ----------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// inclusive product scan across the warp
__device__ __forceinline__ float warp_scan_mul(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { float t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v *= t; }
  return v;
}
__device__ __forceinline__ float warp_scan_add(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { float t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += t; }
  return v;
}
__device__ __forceinline__ float sigmoidf_acc(float x) { return 1.0f / (1.0f + expf(-x)); }

}  // namespace nb
