// train_step.cuh -- the two ends of the optimisation step around the backward (SURVEY 8f rank 2):
//   mse_seed_kernel  : img2mse (run_nerf_helpers.py:9, used at run_nerf.py:764-772): loss += mean((rgb - target)^2) over N x 3
//                      and the gradient seed dL/drgb = 2 (rgb - target) / (3 N) * grad_scale in one pass
//   adam_flat_kernel : torch.optim.Adam(lr, betas=(0.9, 0.999)) (run_nerf.py:207, :776) over ONE flat fp32 buffer holding
//                      every parameter (the buffer the gradient all-reduce also uses), with the reference's exponential
//                      learning-rate decay (run_nerf.py:778-783) evaluated on the device from the step counter
#pragma once
#include "common.cuh"

namespace nb {

// state[0] = loss accumulator (fp32), state[1] = optimizer step count (as float), state[2] = learning rate used last
// ONE block: each thread sums its strided elements in order, then the warps and the block add up in a fixed order, so that the
// loss is the same bits on every run (no atomics).  A batch is a few thousand rays: one block streams it in microseconds.
constexpr int MSE_THREADS = 1024;
__global__ void __launch_bounds__(MSE_THREADS) mse_seed_kernel(const float* __restrict__ rgb, const float* __restrict__ target, long long n3,
                                                             float inv_n3, float grad_scale, float* __restrict__ g, float* __restrict__ loss) {
  __shared__ float s_warp[MSE_THREADS / 32];
  float s = 0.f;
  for (long long i = threadIdx.x; i < n3; i += MSE_THREADS) {
    const float d = rgb[i] - target[i];
    s = fmaf(d, d, s);
    g[i] = 2.0f * d * inv_n3 * grad_scale;
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < MSE_THREADS / 32; ++w) t += s_warp[w];
    *loss += t * inv_n3;
  }
}

// Adam step t = state[1] + 1 on n parameters.  lr_t = lr0 * decay_rate^((t - 2) / decay_steps) for t >= 2, lr0 for t = 1:
// the reference updates the rate AFTER optimizer.step() from global_step before its increment (run_nerf.py:776-784, :872)
__global__ void adam_flat_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                 long long n, const float* __restrict__ state, float lr0, float decay_rate, float decay_steps,
                                 float b1, float b2, float eps, float grad_mul) {
  const float t = state[1] + 1.0f;
  const float lr = (t >= 2.0f && decay_steps > 0.f) ? lr0 * powf(decay_rate, (t - 2.0f) / decay_steps) : lr0;
  const float bc1 = 1.0f - powf(b1, t), bc2 = 1.0f - powf(b2, t);
  const float step_size = lr / bc1, inv_sqrt_bc2 = rsqrtf(bc2);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float gi = g[i] * grad_mul;
    const float mi = b1 * m[i] + (1.0f - b1) * gi;
    const float vi = b2 * v[i] + (1.0f - b2) * gi * gi;
    m[i] = mi; v[i] = vi;
    p[i] -= step_size * mi / (sqrtf(vi) * inv_sqrt_bc2 + eps);
  }
}
__global__ void adam_advance_kernel(float* __restrict__ state, float lr0, float decay_rate, float decay_steps) {
  const float t = state[1] + 1.0f;
  state[1] = t;
  state[2] = (t >= 2.0f && decay_steps > 0.f) ? lr0 * powf(decay_rate, (t - 2.0f) / decay_steps) : lr0;
}

}  // namespace nb
