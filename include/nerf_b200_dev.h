/*
 * nerf_b200_dev.h -- bring-up self-tests and micro-benchmarks (libnerf_b200_dev.so).  NOT part of the drop-in
 * boundary: nothing in the product path calls these; tests/test_gpu_units.py and tools/*_probe.py do.
 */
#ifndef NERF_B200_DEV_H_
#define NERF_B200_DEV_H_
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif
const char* nerf_b200_dev_last_error(void);
/* out[128,N] = fp16(A[128,K]) * fp16(W[N,K])^T with fp32 accumulation through the operand layouts / descriptors
 * of the fused pass (K % 32 == 0, K <= 256, N in {128,256}); scratch >= N*K*2 bytes. */
int nerf_b200_selftest_gemm(const float* A, const float* W, int K, int N, float* out, void* scratch,
                            size_t scratch_bytes, void* stream);
/* out[256,256] = fp16(X[128,256])^T * fp16(Y[128,256]): both operands read as MN-major SWIZZLE_128B tiles straight
 * from the activation layout (lbo = 16384, sbo = 1024) -- the encoding the weight-gradient kernel relies on. */
int nerf_b200_selftest_gemm_tn(const float* X, const float* Y, float* out, int lbo_bytes, int sbo_bytes, void* stream);
/* stream `bytes` of HBM: mode 0 read src, 1 write dst, 2 copy src -> dst; plain 16-byte loads/stores, nblocks x 512 threads */
/* one CTA per SM streams its own bytes_per_cta of `buf`: mode 0 cp.async.bulk g2s ring, 1 cp.async 16 B ring, 2 cp.async.bulk s2g,
 * 3 st.global.v4, 4 ld.global.v4; scatter != 0: the chunks of a region are visited in a strided order; out[nblocks + 1] int64 = cycles per CTA */
int nerf_b200_debug_dram_stream(void* buf, size_t bytes_per_cta, int chunk, int stages, int mode, int nblocks, int scatter, void* out_i64, void* stream);
/* the same; shared_bytes != 0 (mode 0): every CTA streams the first shared_bytes of buf cyclically (L2-resident), bytes_per_cta in all */
int nerf_b200_debug_l2_stream(void* buf, size_t bytes_per_cta, size_t shared_bytes, int chunk, int stages, int mode, int nblocks, int scatter, void* out_i64, void* stream);
int nerf_b200_debug_hbm_stream(const void* src, void* dst, size_t bytes, int mode, int nblocks, void* stream);
#ifdef __cplusplus
}
#endif
#endif
