// bwd_simt.cuh -- exact-mode (fp32 CUDA-core) backward of one network pass: dL/dtheta given dL/drgb_map.
//
// Replaces autograd's backward through run_nerf.py:381-386 / :397-403 (SURVEY 3.5): the pass is
// recomputed in fp32 with saved activations (mlp_simt_kernel, save mode), the compositing adjoint
// (SURVEY App. E) gives dL/draw, and the MLP is walked backwards with two generic fp32 GEMMs
// (dgrad: C = A B, wgrad: C += A^T B reduced over all sample rows), a ReLU-mask and a column-sum
// kernel.  No gradient flows to rays / z (run_nerf.py:394, SURVEY 3.5).  Sums split over blocks are written as fp32 partials
// and added in block order (sum_partials_kernel): no float atomics, the same bits on every run.
// The tensor-core path (bwd_wg.cuh) is the default; this one serves exact mode and networks without view directions.
#pragma once
#include "common.cuh"

namespace nb {

constexpr int GT = 64, GK = 16;   // GEMM tile: 64 x 64 outputs, K step 16, 256 threads x (4 x 4)

// C[M,N] (ldc) = (beta ? C : 0) + A[M,K] (lda) * B[K,N] (ldb)        -- dgrad
__global__ void __launch_bounds__(256) sgemm_nn_kernel(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb,
                                                      float* __restrict__ C, int ldc, long long M, int N, int K, int beta) {
  __shared__ float sA[GK][GT + 4], sB[GK][GT + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const long long m0 = (long long)blockIdx.x * GT;
  const int n0 = blockIdx.y * GT;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += GK) {
    for (int i = threadIdx.x; i < GT * GK; i += 256) {
      int r = i / GK, k = i % GK;                     // A tile: [64 rows][16 k], k contiguous in memory
      long long m = m0 + r;
      sA[k][r] = (m < M && k0 + k < K) ? A[m * lda + k0 + k] : 0.0f;
      int kk = i / GT, c = i % GT;                    // B tile: [16 k][64 n], n contiguous
      sB[kk][c] = (k0 + kk < K && n0 + c < N) ? B[(size_t)(k0 + kk) * ldb + n0 + c] : 0.0f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < GK; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = sA[k][ty * 4 + i]; b[i] = sB[k][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    long long m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int n = n0 + tx * 4 + j;
      if (n < N) { float* c = C + m * ldc + n; *c = (beta ? *c : 0.0f) + acc[i][j]; }
    }
  }
}

// C[K1,N] (ldc) += A[M,K1]^T (lda) * B[M,N] (ldb), reduction over the M sample rows, split across
// blockIdx.z slabs of `rows_per_slab` rows: with one slab the tile adds into C, else slab z writes part[z][K1][N]
// (sum_partials_kernel adds the slabs in order).   -- wgrad
__global__ void __launch_bounds__(256) sgemm_tn_kernel(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb,
                                                      float* __restrict__ C, int ldc, long long M, int K1, int N, int rows_per_slab,
                                                      float* __restrict__ part) {
  __shared__ float sA[GK][GT + 4], sB[GK][GT + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int i0 = blockIdx.x * GT, n0 = blockIdx.y * GT;
  const long long mb = (long long)blockIdx.z * rows_per_slab;
  const long long me = (mb + rows_per_slab < M) ? mb + rows_per_slab : M;
  float acc[4][4] = {};
  for (long long m0 = mb; m0 < me; m0 += GK) {
    for (int i = threadIdx.x; i < GT * GK; i += 256) {
      int mm = i / GT, c = i % GT;                    // both tiles: [16 rows][64 cols], cols contiguous
      long long m = m0 + mm;
      sA[mm][c] = (m < me && i0 + c < K1) ? A[m * lda + i0 + c] : 0.0f;
      sB[mm][c] = (m < me && n0 + c < N) ? B[m * ldb + n0 + c] : 0.0f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < GK; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = sA[k][ty * 4 + i]; b[i] = sB[k][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int r = i0 + ty * 4 + i;
    if (r >= K1) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      if (part) part[((size_t)blockIdx.z * K1 + r) * N + n] = acc[i][j];
      else C[(size_t)r * ldc + n] += acc[i][j];
    }
  }
}

// d[m, c] *= (h[m, c] > 0)   (ReLU backward, in place), and colsum[c] += sum_m d[m, c]  (bias gradient): with one row block
// straight into colsum, else block x writes part[x][C] (sum_partials_kernel adds the blocks in order)
__global__ void relu_mask_colsum_kernel(float* __restrict__ d, int ldd, const float* __restrict__ h, int ldh,
                                        long long M, int C, float* __restrict__ colsum, int rows_per_block, float* __restrict__ part) {
  const int c = blockIdx.y * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const long long m0 = (long long)blockIdx.x * rows_per_block;
  const long long m1 = (m0 + rows_per_block < M) ? m0 + rows_per_block : M;
  float s = 0.0f;
  for (long long m = m0; m < m1; ++m) {
    float v = d[m * ldd + c];
    if (h != nullptr) { v = (h[m * ldh + c] > 0.0f) ? v : 0.0f; d[m * ldd + c] = v; }
    s += v;
  }
  if (part) part[(size_t)blockIdx.x * C + c] = s;
  else if (colsum) colsum[c] += s;
}

// dst[r][c] (ld) += sum_p part[p][r][c], p = 0, 1, ... in order
__global__ void sum_partials_kernel(const float* __restrict__ part, int nparts, int rows, int cols, float* __restrict__ dst, int ld) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * cols) return;
  float s = 0.f;
  for (int q = 0; q < nparts; ++q) s += part[(size_t)q * rows * cols + idx];
  dst[(size_t)(idx / cols) * ld + idx % cols] += s;
}

// ---- the density gradient dsigma/dx at arbitrary points (nerf_b200_density_gradient) ----
// The chain is the exact backward's (gemm_nn, the ReLU mask); these two kernels are its first and last step.

// dA[m, c] = (h[m, c] > 0) * w_sigma[c]: dsigma / d(pre-activation of the last pts layer), w_sigma the density head's row
__global__ void __launch_bounds__(256) sigma_seed_kernel(const float* __restrict__ h, const float* __restrict__ w_sigma, long long M,
                                                         int W, float* __restrict__ dA) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * W) return;
  dA[i] = h[i] > 0.0f ? w_sigma[i % W] : 0.0f;
}

// grad[m, j] = dsigma/dx_j from d_enc [M, IC] = dsigma/d(encoding) through the encoding's Jacobian (run_nerf_helpers.py:36-45,
// columns x, then sin and cos of 2^k x per octave k < L, 3 wide each): d_enc[x_j] + sum_k 2^k (cos(a) d_enc[sin_kj] -
// sin(a) d_enc[cos_kj]), a = 2^k x_j formed as mlp_simt_kernel forms it.  Octaves are added in order: the same bits every run.
__global__ void __launch_bounds__(256) enc_jacobian_kernel(const float* __restrict__ d_enc, int IC, int L, const float* __restrict__ pts,
                                                           long long M, float* __restrict__ grad) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const float* d = d_enc + m * IC;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const float x = pts[m * 3 + j];
    float g = d[j];
    for (int k = 0; k < L; ++k) {
      const float s = exp2f((float)k), a = __fmul_rn(x, s);
      const float t = __fmaf_rn(cosf(a), d[3 + 6 * k + j], -__fmul_rn(sinf(a), d[6 + 6 * k + j]));
      g = __fmaf_rn(s, t, g);
    }
    grad[m * 3 + j] = g;
  }
}

// activations saved by the exact forward (row-major fp32), all optional
struct SimtSave {
  float* enc;    // [M, IC]
  float* encv;   // [M, ICV]  (per-row copy of the ray's view encoding)
  float* h;      // [D][M, W] post-ReLU outputs of pts_linears
  float* feat;   // [M, W]    feature_linear output
  float* hv;     // [M, W/2]  post-ReLU views layer
};

static inline size_t bwd_floats_per_row(const NerfNetParams& n) {
  // enc + encv + h[D] + feat + hv + raw + d_raw + dh ping/pong + d_hv
  return (size_t)n.input_ch + n.input_ch_views + (size_t)n.D * n.W + n.W + n.W / 2 + 4 + 4 + 2 * (size_t)n.W + n.W / 2;
}

}  // namespace nb
