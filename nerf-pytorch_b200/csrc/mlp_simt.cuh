// mlp_simt.cuh -- exact-mode (fp32 CUDA-core) run_network: encode + NeRF.forward -> raw.
// Mirrors run_nerf.py:37-51 and run_nerf_helpers.py:96-119 with fp32 FMA accumulation.  It is the
// validation / "exact" path (NERF_B200_PREC_FP32); the production path is fused_wg.cuh.
#pragma once
#include "common.cuh"
#include "bwd_simt.cuh"

namespace nb {

constexpr int SIMT_ROWS = 32;      // sample rows per CTA
constexpr int SIMT_THREADS = 256;  // one thread per output column (W <= 256)

struct SimtSmem {
  // activations are stored transposed [k][row] so that a thread reads 4 rows per LDS.128 broadcast
};

// acc[r] += sum_k in[k][r] * w[n][k]  for k in [0,K)
__device__ __forceinline__ void simt_dot(float (&acc)[SIMT_ROWS], const float* __restrict__ w_row, int K,
                                         const float* s_in /*[K][SIMT_ROWS]*/) {
  for (int k = 0; k < K; ++k) {
    const float w = __ldg(w_row + k);
    const float4* in4 = reinterpret_cast<const float4*>(s_in + k * SIMT_ROWS);
#pragma unroll
    for (int r4 = 0; r4 < SIMT_ROWS / 4; ++r4) {
      float4 v = in4[r4];
      acc[r4 * 4 + 0] = fmaf(v.x, w, acc[r4 * 4 + 0]);
      acc[r4 * 4 + 1] = fmaf(v.y, w, acc[r4 * 4 + 1]);
      acc[r4 * 4 + 2] = fmaf(v.z, w, acc[r4 * 4 + 2]);
      acc[r4 * 4 + 3] = fmaf(v.w, w, acc[r4 * 4 + 3]);
    }
  }
}

__device__ __forceinline__ void simt_store(const float (&acc)[SIMT_ROWS], float* s_out_row, bool relu) {
#pragma unroll
  for (int r = 0; r < SIMT_ROWS; ++r) s_out_row[r] = relu ? fmaxf(acc[r], 0.0f) : acc[r];
}

// pts [M,3] (M = N*S), viewdirs [N,3] or NULL, raw [M,4]
__global__ void __launch_bounds__(SIMT_THREADS)
mlp_simt_kernel(const float* __restrict__ pts, const float* __restrict__ viewdirs, int dir_stride, long long M, int S,
                NerfNetParams net, int L, int Lv, float* __restrict__ raw, SimtSave sv) {
  extern __shared__ __align__(16) float smem[];
  const int W = net.W, IC = net.input_ch, ICV = net.input_ch_views;
  float* s_enc = smem;                                  // [IC][ROWS]
  float* s_encv = s_enc + IC * SIMT_ROWS;               // [ICV][ROWS]
  float* s_h0 = s_encv + ICV * SIMT_ROWS;               // [W][ROWS]
  float* s_h1 = s_h0 + W * SIMT_ROWS;                   // [W][ROWS]
  const int tid = threadIdx.x;
  const long long row0 = (long long)blockIdx.x * SIMT_ROWS;
  // save a [C][ROWS] shared-memory block as rows of a row-major [M, C] global matrix (training only)
  auto save_rows = [&](float* dst, const float* s_src, int C) {
    if (dst == nullptr) return;
    for (int i = tid; i < C * SIMT_ROWS; i += SIMT_THREADS) {
      int r = i / C, c = i - r * C;
      if (row0 + r < M) dst[(row0 + r) * C + c] = s_src[c * SIMT_ROWS + r];
    }
  };

  // ---- positional encoding (run_nerf_helpers.py:36-45) ----
  for (int i = tid; i < IC * SIMT_ROWS; i += SIMT_THREADS) {
    int c = i / SIMT_ROWS, r = i % SIMT_ROWS;
    long long m = row0 + r;
    float v = 0.0f;
    if (m < M) {
      if (c < 3) v = pts[m * 3 + c];
      else { int f = (c - 3) / 6, q = (c - 3) % 6; float a = __fmul_rn(pts[m * 3 + (q % 3)], exp2f((float)f)); v = (q < 3) ? sinf(a) : cosf(a); }
    }
    s_enc[i] = v;
  }
  for (int i = tid; i < ICV * SIMT_ROWS; i += SIMT_THREADS) {
    int c = i / SIMT_ROWS, r = i % SIMT_ROWS;
    long long m = row0 + r;
    float v = 0.0f;
    if (m < M) {
      long long n = m / S;
      if (c < 3) v = viewdirs[n * dir_stride + c];
      else { int f = (c - 3) / 6, q = (c - 3) % 6; float a = __fmul_rn(viewdirs[n * dir_stride + (q % 3)], exp2f((float)f)); v = (q < 3) ? sinf(a) : cosf(a); }
    }
    s_encv[i] = v;
  }
  __syncthreads();
  save_rows(sv.enc, s_enc, IC);
  save_rows(sv.encv, s_encv, ICV);

  float acc[SIMT_ROWS];
  float* h_in = s_h0;
  float* h_out = s_h1;
  const int n = tid;
  // ---- pts_linears (run_nerf_helpers.py:99-103) ----
  for (int i = 0; i < net.D; ++i) {
    const bool after_skip = (i > 0) && (i - 1 == net.skip);
    const int K = (i == 0) ? IC : (after_skip ? W + IC : W);
    if (n < W) {
      const float b = net.pts_b[i][n];
#pragma unroll
      for (int r = 0; r < SIMT_ROWS; ++r) acc[r] = b;
      const float* wr = net.pts_w[i] + (size_t)n * K;
      if (i == 0) simt_dot(acc, wr, IC, s_enc);
      else if (after_skip) { simt_dot(acc, wr, IC, s_enc); simt_dot(acc, wr + IC, W, h_in); }   // cat([input_pts, h])
      else simt_dot(acc, wr, W, h_in);
      simt_store(acc, h_out + n * SIMT_ROWS, true);
    }
    __syncthreads();
    save_rows(sv.h ? sv.h + (size_t)i * M * W : nullptr, h_out, W);
    float* t = h_in; h_in = h_out; h_out = t;
  }
  // h_in now holds h of the last pts layer
  if (net.use_viewdirs) {
    // alpha (:106): threads 0..31 -> one row each; kept in a register until the final store
    float alpha = 0.0f;
    if (tid < SIMT_ROWS) {
      alpha = net.alpha_b[0];
      for (int k = 0; k < W; ++k) alpha = fmaf(h_in[k * SIMT_ROWS + tid], __ldg(net.alpha_w + k), alpha);
    }
    // feature (:107), no activation
    if (n < W) {
      const float b = net.feature_b[n];
#pragma unroll
      for (int r = 0; r < SIMT_ROWS; ++r) acc[r] = b;
      simt_dot(acc, net.feature_w + (size_t)n * W, W, h_in);
      simt_store(acc, h_out + n * SIMT_ROWS, false);
    }
    __syncthreads();
    save_rows(sv.feat, h_out, W);
    // views_linears[0] on cat([feature, input_views]) (:108-112)
    const int W2 = W / 2;
    if (n < W2) {
      const float b = net.views_b[n];
#pragma unroll
      for (int r = 0; r < SIMT_ROWS; ++r) acc[r] = b;
      const float* wr = net.views_w + (size_t)n * (W + ICV);
      simt_dot(acc, wr, W, h_out);
      simt_dot(acc, wr + W, ICV, s_encv);
      simt_store(acc, h_in + n * SIMT_ROWS, true);       // h_in is free (alpha/feature already read) ...
    }
    __syncthreads();
    save_rows(sv.hv, h_in, W2);
    // rgb (:114) and output cat([rgb, alpha]) (:115)
    if (tid < SIMT_ROWS) {
      long long m = row0 + tid;
      float o[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float a = net.rgb_b[c];
        for (int k = 0; k < W2; ++k) a = fmaf(h_in[k * SIMT_ROWS + tid], __ldg(net.rgb_w + c * W2 + k), a);
        o[c] = a;
      }
      if (m < M) reinterpret_cast<float4*>(raw)[m] = make_float4(o[0], o[1], o[2], alpha);
    }
  } else {
    // output_linear (:117): only the first four channels are ever read (run_nerf.py:187 note)
    if (tid < SIMT_ROWS) {
      long long m = row0 + tid;
      float o[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        float a = net.output_b[c];
        for (int k = 0; k < W; ++k) a = fmaf(h_in[k * SIMT_ROWS + tid], __ldg(net.output_w + c * W + k), a);
        o[c] = a;
      }
      if (m < M) reinterpret_cast<float4*>(raw)[m] = make_float4(o[0], o[1], o[2], o[3]);
    }
  }
}

static inline size_t simt_smem_bytes(const NerfNetParams& net) {
  return sizeof(float) * SIMT_ROWS * (size_t)(net.input_ch + net.input_ch_views + 2 * net.W);
}

}  // namespace nb
