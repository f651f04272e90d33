// capi_dev.cu -- extern "C" entry points of libnerf_b200_dev.so: self-tests and micro-benchmarks used by tests/ and
// tools/ during bring-up and profiling.  Not part of the product ABI (include/nerf_b200.h); declared in
// include/nerf_b200_dev.h.
#include <stdarg.h>
#include "common.cuh"
#include "dev_kernels.cuh"
#include "../../include/nerf_b200_dev.h"

namespace nb {
thread_local char g_err[512] = {0};
long long g_launches = 0;
int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
static int smem_optin(const void* fn, size_t bytes) {
  NB_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return 0;
}
}  // namespace nb

using namespace nb;

extern "C" {

const char* nerf_b200_dev_last_error(void) { return g_err; }

int nerf_b200_selftest_gemm_tn(const float* X, const float* Y, float* out, int lbo_bytes, int sbo_bytes, void* stream) {
  NB_CHECK_ARG(X && Y && out, "null pointer");
  NB_CHECK_ARG(lbo_bytes >= 0 && sbo_bytes >= 0 && lbo_bytes % 16 == 0 && sbo_bytes % 16 == 0, "lbo / sbo must be multiples of 16 bytes");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int sm = 131072;
  if (int rc = smem_optin((const void*)selftest_gemm_tn_kernel, sm)) return rc;
  selftest_gemm_tn_kernel<<<1, 128, sm, st>>>(X, Y, out, (uint32_t)lbo_bytes, (uint32_t)sbo_bytes);
  NB_LAUNCH_OK("selftest_gemm_tn_kernel");
  return 0;
}

int nerf_b200_selftest_gemm(const float* A, const float* W, int K, int N, float* out, void* scratch, size_t scratch_bytes, void* stream) {
  NB_CHECK_ARG(A && W && out && scratch, "NULL pointer");
  NB_CHECK_ARG(K % 32 == 0 && K >= 32 && K <= 256 && (N == 128 || N == 256), "bad K/N");
  NB_CHECK_ARG(scratch_bytes >= (size_t)N * K * 2, "scratch too small");
  cudaStream_t st = (cudaStream_t)stream;
  PackJob job;
  job.n = 0;
  for (int c = 0; c < K / 32; ++c) { PackChunk& pc = job.c[job.n++]; pc.src = W; pc.sn = K; pc.sk = 1; pc.k0 = 32 * c; pc.kvalid = 32; pc.nrows = N; pc.dst_off = (unsigned)c * N * 64; }
  dim3 grid(4, job.n);
  pack_chunks_kernel<<<grid, 256, 0, st>>>(job, static_cast<uint8_t*>(scratch));
  NB_LAUNCH_OK("pack_chunks_kernel");
  const size_t sm = 65536 + 131072 + 64;
  if (int rc = smem_optin((const void*)selftest_gemm_kernel, sm)) return rc;
  selftest_gemm_kernel<<<1, 256, sm, st>>>(A, static_cast<const uint8_t*>(scratch), K, N, out);
  NB_LAUNCH_OK("selftest_gemm_kernel");
  return 0;
}

int nerf_b200_debug_hbm_stream(const void* src, void* dst, size_t bytes, int mode, int nblocks, void* stream) {
  NB_CHECK_ARG(bytes % 16 == 0 && mode >= 0 && mode <= 2 && nblocks > 0, "bad arguments");
  NB_CHECK_ARG((mode == 1 || src) && (mode == 0 || dst), "NULL pointer");
  static uint4* sink = nullptr;
  if (!sink) NB_CUDA(cudaMalloc(&sink, 64));
  hbm_stream_kernel<<<nblocks, 512, 0, (cudaStream_t)stream>>>(static_cast<const uint4*>(src), static_cast<uint4*>(dst), bytes / 16, mode, sink);
  NB_LAUNCH_OK("hbm_stream_kernel");
  return 0;
}

int nerf_b200_debug_dram_stream(void* buf, size_t bytes_per_cta, int chunk, int stages, int mode, int nblocks, int scatter, void* out_i64, void* stream) {
  return nerf_b200_debug_l2_stream(buf, bytes_per_cta, 0, chunk, stages, mode, nblocks, scatter, out_i64, stream);
}

int nerf_b200_debug_l2_stream(void* buf, size_t bytes_per_cta, size_t shared_bytes, int chunk, int stages, int mode, int nblocks, int scatter, void* out_i64, void* stream) {
  NB_CHECK_ARG(buf && out_i64 && nblocks > 0 && mode >= 0 && mode <= 4, "bad arguments");
  NB_CHECK_ARG(chunk >= 1024 && chunk % 1024 == 0 && stages >= 1 && stages <= 8 && (size_t)stages * chunk <= 196608, "ring too large");
  NB_CHECK_ARG(bytes_per_cta % (size_t)chunk == 0, "bytes_per_cta must be a multiple of chunk");
  NB_CHECK_ARG(shared_bytes == 0 || (mode == 0 && shared_bytes % (size_t)chunk == 0), "a shared region is streamed by mode 0, in whole chunks");
  const size_t sm = (size_t)stages * chunk + 512 + 1024;
  if (int rc = smem_optin((const void*)dram_stream_probe_kernel, sm)) return rc;
  dram_stream_probe_kernel<<<nblocks, DSP_THREADS, sm, (cudaStream_t)stream>>>(static_cast<uint8_t*>(buf), (unsigned long long)bytes_per_cta, chunk, stages, mode,
                                                                              static_cast<long long*>(out_i64), scatter, (unsigned long long)shared_bytes);
  NB_LAUNCH_OK("dram_stream_probe_kernel");
  return 0;
}

}  // extern "C"
