// small_kernels.cuh -- the exactly-checkable per-ray kernels of the NeRF hot path:
//   Embedder.embed, coarse z sampling, raw2outputs (+adjoint), sample_pdf, hierarchical z merge.
// All fp32, one warp per ray where a ray-wide scan is needed.  Non-fused mul/add intrinsics are
// used where the reference rounds twice (torch evaluates a*b+c as two ops), so z values and
// sample positions agree with the reference to the last bit wherever the op order allows.
#pragma once
#include "common.cuh"

namespace nb {

// ---------------------------------------------------------------------------------------------
// Embedder.embed  (run_nerf_helpers.py:36-45): out[m] = [x, sin(2^0 x), cos(2^0 x), ...]
// ---------------------------------------------------------------------------------------------
__global__ void embed_kernel(const float* __restrict__ x, long long M, int L, float* __restrict__ out) {
  const int C = 3 + 6 * L;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * C) return;
  long long m = i / C;
  int c = (int)(i - m * C);
  float v;
  if (c < 3) {
    v = x[m * 3 + c];
  } else {
    int f = (c - 3) / 6, r = (c - 3) % 6;
    float a = __fmul_rn(x[m * 3 + (r % 3)], exp2f((float)f));   // exact power-of-two scaling (:32)
    v = (r < 3) ? sinf(a) : cosf(a);
  }
  out[i] = v;
}

// ---------------------------------------------------------------------------------------------
// coarse z sampling  (run_nerf.py:357-379)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float coarse_z_at(float near, float far, float t, int lindisp) {
  float omt = __fsub_rn(1.0f, t);
  if (!lindisp) return __fadd_rn(__fmul_rn(near, omt), __fmul_rn(far, t));                   // :359
  float a = __fmul_rn(__fdiv_rn(1.0f, near), omt), b = __fmul_rn(__fdiv_rn(1.0f, far), t);
  return __fdiv_rn(1.0f, __fadd_rn(a, b));                                                    // :361
}

__global__ void coarse_z_kernel(const float* __restrict__ rays, int ray_stride,
                                const float* __restrict__ t_vals, const float* __restrict__ t_rand,
                                long long N, int S, int lindisp, float* __restrict__ z_out) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * S) return;
  long long n = i / S;
  int s = (int)(i - n * S);
  float near = rays[n * ray_stride + 6], far = rays[n * ray_stride + 7];
  float z = coarse_z_at(near, far, t_vals[s], lindisp);
  if (t_rand != nullptr) {
    float zl = (s > 0) ? coarse_z_at(near, far, t_vals[s - 1], lindisp) : z;
    float zu = (s < S - 1) ? coarse_z_at(near, far, t_vals[s + 1], lindisp) : z;
    float lower = (s > 0) ? __fmul_rn(0.5f, __fadd_rn(z, zl)) : z;                           // :367-369
    float upper = (s < S - 1) ? __fmul_rn(0.5f, __fadd_rn(zu, z)) : z;
    z = __fadd_rn(lower, __fmul_rn(__fsub_rn(upper, lower), t_rand[i]));                      // :379
  }
  z_out[i] = z;
}

// ---------------------------------------------------------------------------------------------
// ray batch construction of render()  (run_nerf.py:95-123): optional pinhole ray generation
// (get_rays, run_nerf_helpers.py:153-162), view-direction normalisation (:108), optional NDC warp
// (ndc_rays, run_nerf_helpers.py:175-192) and packing to [N, 8|11] = o d near far [viewdir].
// Every product/sum is rounded separately, in the reference's order.
// ---------------------------------------------------------------------------------------------
struct PackRaysArgs {
  const float* rays_o; const float* rays_d;     // [N,3] each, or NULL -> generate from the camera
  const float* view_src;                        // [N,3] directions for viewdirs, or NULL -> rays_d
  int H, W; float fx, fy, cx, cy; float c2w[12];
  long long N, pixel0;
  const long long* pixel_index;                 // [N] pixel ids (row-major j * W + i) or NULL -> pixel0 + n
  int ndc, use_viewdirs, stride;
  float near, far, ndc_cw, ndc_ch;              // ndc_cw = -1/(W/(2 focal)), ndc_ch = -1/(H/(2 focal)) (host double -> float)
};

// row n of the batch -> out + n * stride
__device__ __forceinline__ void pack_ray_row(const PackRaysArgs& a, long long n, float* __restrict__ out) {
  float o[3], d[3];
  if (a.rays_d != nullptr) {
#pragma unroll
    for (int k = 0; k < 3; ++k) { o[k] = a.rays_o[n * 3 + k]; d[k] = a.rays_d[n * 3 + k]; }
  } else {
    const long long pix = a.pixel_index ? a.pixel_index[n] : a.pixel0 + n;
    const float i = (float)(pix % a.W), j = (float)(pix / a.W);                       // :154-156 (i along W, j along H)
    const float dir[3] = {__fdiv_rn(__fsub_rn(i, a.cx), a.fx), -__fdiv_rn(__fsub_rn(j, a.cy), a.fy), -1.0f};   // :157
#pragma unroll
    for (int k = 0; k < 3; ++k) {                                                     // :159 sum(dirs[..., None, :] * c2w[:3,:3], -1)
      d[k] = __fadd_rn(__fadd_rn(__fmul_rn(dir[0], a.c2w[4 * k]), __fmul_rn(dir[1], a.c2w[4 * k + 1])), __fmul_rn(dir[2], a.c2w[4 * k + 2]));
      o[k] = a.c2w[4 * k + 3];                                                        // :161
    }
  }
  float* r = out + n * a.stride;
  if (a.use_viewdirs) {
    float v[3];
    if (a.view_src != nullptr) { v[0] = a.view_src[n * 3]; v[1] = a.view_src[n * 3 + 1]; v[2] = a.view_src[n * 3 + 2]; }
    else { v[0] = d[0]; v[1] = d[1]; v[2] = d[2]; }
    const float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(v[0], v[0]), __fmul_rn(v[1], v[1])), __fmul_rn(v[2], v[2])));
    r[8] = __fdiv_rn(v[0], nrm); r[9] = __fdiv_rn(v[1], nrm); r[10] = __fdiv_rn(v[2], nrm);   // run_nerf.py:108
  }
  if (a.ndc) {                                                                        // ndc_rays(H, W, focal, near=1.)
    const float t = __fdiv_rn(-__fadd_rn(1.0f, o[2]), d[2]);
#pragma unroll
    for (int k = 0; k < 3; ++k) o[k] = __fadd_rn(o[k], __fmul_rn(t, d[k]));
    const float o0 = __fdiv_rn(__fmul_rn(a.ndc_cw, o[0]), o[2]), o1 = __fdiv_rn(__fmul_rn(a.ndc_ch, o[1]), o[2]);
    const float o2 = __fadd_rn(1.0f, __fdiv_rn(2.0f, o[2]));
    const float d0 = __fmul_rn(a.ndc_cw, __fsub_rn(__fdiv_rn(d[0], d[2]), __fdiv_rn(o[0], o[2])));
    const float d1 = __fmul_rn(a.ndc_ch, __fsub_rn(__fdiv_rn(d[1], d[2]), __fdiv_rn(o[1], o[2])));
    const float d2 = __fdiv_rn(-2.0f, o[2]);
    o[0] = o0; o[1] = o1; o[2] = o2; d[0] = d0; d[1] = d1; d[2] = d2;
  }
  r[0] = o[0]; r[1] = o[1]; r[2] = o[2]; r[3] = d[0]; r[4] = d[1]; r[5] = d[2]; r[6] = a.near; r[7] = a.far;
}
__global__ void pack_rays_kernel(PackRaysArgs a, float* __restrict__ out) {
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n < a.N) pack_ray_row(a, n, out);
}

// to8b (run_nerf_helpers.py:11: (255 * clip(x, 0, 1)).astype(uint8)) on the device, for render_path-style image output
__global__ void to8b_kernel(const float* __restrict__ x, long long n, uint8_t* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = x[i];
  out[i] = (uint8_t)(255.0f * fminf(fmaxf(v, 0.0f), 1.0f));      // NaN -> fmaxf gives 0, like np.clip + astype on most platforms
}

// pts = rays_o + rays_d * z  (run_nerf.py:381), exact-mode helper
__global__ void pts_kernel(const float* __restrict__ rays, int ray_stride, const float* __restrict__ z_vals,
                           long long M, int S, float* __restrict__ pts) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const float* r = rays + (i / S) * ray_stride;
  const float z = z_vals[i];
  pts[i * 3 + 0] = __fadd_rn(r[0], __fmul_rn(r[3], z));
  pts[i * 3 + 1] = __fadd_rn(r[1], __fmul_rn(r[4], z));
  pts[i * 3 + 2] = __fadd_rn(r[2], __fmul_rn(r[5], z));
}

// ---------------------------------------------------------------------------------------------
// raw2outputs  (run_nerf.py:262-305), one warp per ray
// ---------------------------------------------------------------------------------------------
struct CompositeAcc { float r, g, b, depth, acc, T; };

// Composite up to 32 consecutive samples held one per lane; carries transmittance in `a.T`.
__device__ __forceinline__ float composite_chunk(float alpha, float cr, float cg, float cb, float z,
                                                 bool valid, int lane, CompositeAcc& a) {
  float q = valid ? __fadd_rn(__fsub_rn(1.0f, alpha), 1e-10f) : 1.0f;                         // :295
  float incl = warp_scan_mul(q, lane);
  float excl = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) excl = 1.0f;
  float T = a.T * excl;
  float w = valid ? alpha * T : 0.0f;
  a.r += w * cr; a.g += w * cg; a.b += w * cb; a.depth += w * z; a.acc += w;
  a.T *= __shfl_sync(0xffffffffu, incl, 31);
  return w;
}

__device__ __forceinline__ float disp_from(float depth, float acc) {
  float ratio = depth / acc;                                   // 0/0 -> NaN, like the reference
  float m = (ratio != ratio) ? ratio : fmaxf(1e-10f, ratio);   // torch.max propagates NaN (:299)
  return 1.0f / m;
}

__global__ void raw2outputs_kernel(const float* __restrict__ raw, const float* __restrict__ z_vals,
                                   const float* __restrict__ rays_d, int d_stride,
                                   const float* __restrict__ noise, long long N, int S, int white_bkgd,
                                   NerfPassOut out) {
  const int lane = threadIdx.x & 31;
  long long n = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (n >= N) return;
  const float dx = rays_d[n * d_stride], dy = rays_d[n * d_stride + 1], dz = rays_d[n * d_stride + 2];
  const float norm = sqrtf(dx * dx + dy * dy + dz * dz);                                      // :280
  CompositeAcc a = {0, 0, 0, 0, 0, 1.0f};
  for (int base = 0; base < S; base += 32) {
    int k = base + lane;
    bool valid = k < S;
    float alpha = 0, cr = 0, cg = 0, cb = 0, z = 0;
    if (valid) {
      float4 r4 = reinterpret_cast<const float4*>(raw)[n * S + k];
      z = z_vals[n * S + k];
      float dist = (k == S - 1) ? 1e10f : __fsub_rn(z_vals[n * S + k + 1], z);               // :277-278
      dist = __fmul_rn(dist, norm);
      float s = r4.w + (noise ? noise[n * S + k] : 0.0f);
      alpha = __fsub_rn(1.0f, expf(-fmaxf(s, 0.0f) * dist));                                  // :275
      cr = sigmoidf_acc(r4.x); cg = sigmoidf_acc(r4.y); cb = sigmoidf_acc(r4.z);             // :282
    }
    float w = composite_chunk(alpha, cr, cg, cb, z, valid, lane, a);
    if (valid && out.weights) out.weights[n * S + k] = w;
  }
  float r = warp_sum(a.r), g = warp_sum(a.g), b = warp_sum(a.b);
  float depth = warp_sum(a.depth), acc = warp_sum(a.acc);
  if (lane == 0) {
    if (white_bkgd) { float bg = 1.0f - acc; r += bg; g += bg; b += bg; }                      // :302-303
    if (out.rgb_map) { out.rgb_map[n * 3] = r; out.rgb_map[n * 3 + 1] = g; out.rgb_map[n * 3 + 2] = b; }
    if (out.disp_map) out.disp_map[n] = disp_from(depth, acc);
    if (out.acc_map) out.acc_map[n] = acc;
    if (out.depth_map) out.depth_map[n] = depth;
  }
}

// Seeds of the compositing adjoint: dL/d(each output of raw2outputs), as in include/nerf_b200.h's NerfOutGrads.  Any
// pointer may be NULL (that output does not reach the loss).  amax: see raw2outputs_bwd_kernel.
struct R2OSeeds {
  const float* rgb;        // [N,3]
  const float* disp;       // [N]
  const float* acc;        // [N]
  const float* depth;      // [N]
  const float* weights;    // [N,S]
  const float* raw;        // [N,S,4]
  unsigned int* amax;      // NULL, or max |effective seed| as a float bit pattern (atomicMax, zeroed by the caller)
};

// NaN-propagating max of |v| (absmax_kernel's rule: non-negative floats order like their bit patterns)
__device__ __forceinline__ float absmax_step(float m, float v) { v = fabsf(v); return (v > m || v != v) ? v : m; }

// Adjoint of raw2outputs w.r.t. raw (SURVEY Appendix E).  One warp per ray, per-warp scratch of 4*S floats in dynamic
// shared memory.  With e_k = dL/dw_k, dL/dalpha_k = T_k e_k - sum_{j>k} w_j e_j / q_k; every seed reaches raw through e_k:
//   rgb:     e_k += sum_c g_c (c_k - off)           (off = 1 with a white background: rgb_map += 1 - acc)
//   acc:     e_k += g_acc          depth: e_k += g_depth z_k          weights: e_k += g_w[k]
//   disp  =  1 / max(1e-10, depth / acc)  (run_nerf.py:299) becomes acc and depth seeds; the ray's depth and acc are
//            RECOMPUTED here from raw with composite_chunk, the order of raw2outputs_kernel.  Like the reference's autograd:
//            no gradient where depth/acc < 1e-10, half of it at equality (torch.max's tie rule), NaN where acc = 0.
//   raw:     added to dL/draw.
// kSeeds = false is the rgb-only adjoint (g.rgb required, everything else ignored): its arithmetic is the one the library
// always had.  kSeeds = true branches on the NULLs; with g.amax it also forms the pass's loss-scale input
//   amax = max( |g_rgb|, |g_acc_eff|, |g_depth_eff z_k|, |g_w|, |g_raw| )   (only over the seeds given)
// which with g_rgb alone equals absmax_kernel's max |g_rgb|.  Rays with acc = 0 under a disp seed are left out of the
// acc / depth terms: their NaN reaches dL/draw only where the density is > 0, and must not reset the whole pass's scale.
template <bool kSeeds>
__global__ void raw2outputs_bwd_kernel(const float* __restrict__ raw, const float* __restrict__ z_vals,
                                       const float* __restrict__ rays_d, int d_stride,
                                       const float* __restrict__ noise, long long N, int S, int white_bkgd,
                                       const R2OSeeds g, float* __restrict__ d_raw) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  long long n = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (n >= N) return;
  float* sT = smem + (size_t)wib * 4 * S;      // T_k e_k
  float* sWE = sT + S;                         // w_k e_k
  float* sQ = sWE + S;                         // q_k
  float* sF = sQ + S;                          // dist * (1-alpha) * [s>0]
  const float dx = rays_d[n * d_stride], dy = rays_d[n * d_stride + 1], dz = rays_d[n * d_stride + 2];
  const float norm = sqrtf(dx * dx + dy * dy + dz * dz);
  const bool has_rgb = !kSeeds || g.rgb != nullptr;
  float gr = 0.f, gg = 0.f, gb = 0.f;
  if (has_rgb) { gr = g.rgb[n * 3]; gg = g.rgb[n * 3 + 1]; gb = g.rgb[n * 3 + 2]; }
  float g_acc = 0.f, g_depth = 0.f, m = 0.f;   // effective per-ray acc / depth seeds; running max for g.amax
  bool disp_nan = false;                       // acc = 0 with a disp seed: g_acc / g_depth are NaN on this ray
  if constexpr (kSeeds) {
    if (g.acc) g_acc = g.acc[n];
    if (g.depth) g_depth = g.depth[n];
    if (g.disp) {
      CompositeAcc a = {0, 0, 0, 0, 0, 1.0f};
      for (int base = 0; base < S; base += 32) {
        int k = base + lane;
        bool valid = k < S;
        float alpha = 0, z = 0;
        if (valid) {
          z = z_vals[n * S + k];
          float dist = (k == S - 1) ? 1e10f : __fsub_rn(z_vals[n * S + k + 1], z);
          dist = __fmul_rn(dist, norm);
          float s = raw[(n * S + k) * 4 + 3] + (noise ? noise[n * S + k] : 0.0f);
          alpha = __fsub_rn(1.0f, expf(-fmaxf(s, 0.0f) * dist));
        }
        composite_chunk(alpha, 0.f, 0.f, 0.f, z, valid, lane, a);
      }
      const float depth = warp_sum(a.depth), acc = warp_sum(a.acc);
      const float ratio = depth / acc;
      const float mx = (ratio != ratio) ? ratio : fmaxf(1e-10f, ratio);
      float g_ratio = -g.disp[n] / (mx * mx);                         // d(1/mx)/dmx
      if (ratio < 1e-10f) g_ratio = 0.f; else if (ratio == 1e-10f) g_ratio *= 0.5f;
      g_depth += g_ratio / acc;
      g_acc -= g_ratio * depth / (acc * acc);
      disp_nan = ratio != ratio;
    }
    if (g.amax) {
      if (has_rgb) { m = absmax_step(m, gr); m = absmax_step(m, gg); m = absmax_step(m, gb); }
      if ((g.acc || g.disp) && !disp_nan) m = absmax_step(m, g_acc);
    }
  }
  float carryT = 1.0f;
  for (int base = 0; base < S; base += 32) {
    int k = base + lane;
    bool valid = k < S;
    float q = 1.0f, alpha = 0, e = 0, f = 0, cr = 0, cg = 0, cb = 0;
    float4 gw4 = make_float4(0.f, 0.f, 0.f, 0.f);                  // dL/draw seed of this sample
    if (valid) {
      float4 r4 = reinterpret_cast<const float4*>(raw)[n * S + k];
      float z = z_vals[n * S + k];
      float dist = (k == S - 1) ? 1e10f : __fsub_rn(z_vals[n * S + k + 1], z);
      dist = __fmul_rn(dist, norm);
      float s = r4.w + (noise ? noise[n * S + k] : 0.0f);
      float oma = expf(-fmaxf(s, 0.0f) * dist);
      alpha = __fsub_rn(1.0f, oma);
      q = __fadd_rn(__fsub_rn(1.0f, alpha), 1e-10f);
      cr = sigmoidf_acc(r4.x); cg = sigmoidf_acc(r4.y); cb = sigmoidf_acc(r4.z);
      float off = white_bkgd ? 1.0f : 0.0f;
      if (has_rgb) e = gr * (cr - off) + gg * (cg - off) + gb * (cb - off);
      if constexpr (kSeeds) {
        if (g.acc || g.disp) e += g_acc;
        if (g.depth || g.disp) {
          const float t = g_depth * z;
          e += t;
          if (g.amax && !disp_nan) m = absmax_step(m, t);
        }
        if (g.weights) {
          const float t = g.weights[n * S + k];
          e += t;
          if (g.amax) m = absmax_step(m, t);
        }
        if (g.raw) {
          gw4 = reinterpret_cast<const float4*>(g.raw)[n * S + k];
          if (g.amax) { m = absmax_step(m, gw4.x); m = absmax_step(m, gw4.y); m = absmax_step(m, gw4.z); m = absmax_step(m, gw4.w); }
        }
      }
      f = (s > 0.0f) ? dist * oma : 0.0f;
    }
    float incl = warp_scan_mul(q, lane);
    float excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 1.0f;
    float T = carryT * excl;
    carryT *= __shfl_sync(0xffffffffu, incl, 31);
    if (valid) {
      float w = alpha * T;
      sT[k] = T * e; sWE[k] = w * e; sQ[k] = q; sF[k] = f;   // sT holds the first term of dL/dalpha
      float* o = d_raw + (n * S + k) * 4;
      if (has_rgb) {
        o[0] = w * gr * cr * (1.0f - cr);
        o[1] = w * gg * cg * (1.0f - cg);
        o[2] = w * gb * cb * (1.0f - cb);
      } else {
        o[0] = 0.f; o[1] = 0.f; o[2] = 0.f;
      }
      if constexpr (kSeeds) {
        if (g.raw) { o[0] += gw4.x; o[1] += gw4.y; o[2] += gw4.z; }
      }
    }
  }
  if constexpr (kSeeds) {
    if (g.amax) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) { const float t = __shfl_xor_sync(0xffffffffu, m, o); m = (t > m || t != t) ? t : m; }
      if (lane == 0) atomicMax(g.amax, __float_as_uint(m));
    }
  }
  __syncwarp();
  // reverse pass: suffix_k = sum_{j>k} w_j e_j
  float carry = 0.0f;
  const int nchunks = (S + 31) / 32;
  for (int c = nchunks - 1; c >= 0; --c) {
    int k = c * 32 + (31 - lane);                     // lane 0 holds the last sample of the chunk
    bool valid = k < S;
    float we = valid ? sWE[k] : 0.0f;
    float incl = warp_scan_add(we, lane);             // sum of we over samples >= k within the chunk
    float suffix = carry + incl - we;
    carry += __shfl_sync(0xffffffffu, incl, 31);
    if (valid) {
      float* o = d_raw + (n * S + k) * 4;
      float dalpha = sT[k] - suffix / sQ[k];
      o[3] = dalpha * sF[k];
      if constexpr (kSeeds) {
        if (disp_nan) {                  // relu's gradient is a select: the NaN reaches only samples with density > 0
          const float s = raw[(n * S + k) * 4 + 3] + (noise ? noise[n * S + k] : 0.0f);
          if (!(s > 0.0f)) o[3] = 0.0f;
        }
        if (g.raw) o[3] += g.raw[(n * S + k) * 4 + 3];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// sample_pdf  (run_nerf_helpers.py:196-239) on per-warp shared-memory rows
// ---------------------------------------------------------------------------------------------
// sum(w + 1e-5) over w = s_w[0..n) (:198-199), rounded exactly as CPU torch's float32 sum(-1) of a contiguous row, so the
// cdf and every sample match the reference to the bit (oracle/resample.py torch_sum states the order).  Warp-uniform result.
//   n < 8:  four accumulators a_k += x[4j+k], the leftover x[4*(n/4)..] into a_0, then ((a_0 + a_1) + a_2) + a_3.
//   n >= 8: the same over 8-wide vectors v_i = x[8i..8i+7] (V = n/8 of them), which is one accumulator per lane here:
//           lane l sums x[32r + l] for r < n/32, with a cascade that moves the running sum into a second accumulator
//           after every 16 rows (the next cascade level needs >= 256 rows, n >= 8192, beyond the accepted sizes);
//           lanes 0-7 add the leftover vectors and then lanes 8-15, 16-23, 24-31 in that order; the total is 0, plus the
//           scalar tail x[8V..n) in order, plus the 8 lanes in order.
__device__ __forceinline__ float torch_row_sum(const float* s_w, int n, int lane) {
  auto x = [&](int i) { return __fadd_rn(s_w[i], 1e-5f); };
  if (n < 8) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    if (n >= 4) { a0 = __fadd_rn(a0, x(0)); a1 = __fadd_rn(a1, x(1)); a2 = __fadd_rn(a2, x(2)); a3 = __fadd_rn(a3, x(3)); }
    for (int i = n & ~3; i < n; ++i) a0 = __fadd_rn(a0, x(i));
    return __fadd_rn(__fadd_rn(__fadd_rn(a0, a1), a2), a3);
  }
  const int V = n >> 3, rows = V >> 2;
  float a0 = 0.f, a1 = 0.f;
  int r = 0;
  for (; r + 16 <= rows; r += 16) {
    for (int k = 0; k < 16; ++k) a0 = __fadd_rn(a0, x(32 * (r + k) + lane));
    a1 = __fadd_rn(a1, a0);
    a0 = 0.f;
  }
  for (; r < rows; ++r) a0 = __fadd_rn(a0, x(32 * r + lane));
  a0 = __fadd_rn(a0, a1);
  if (lane < 8) for (int v = 4 * rows; v < V; ++v) a0 = __fadd_rn(a0, x(8 * v + lane));
  const float p1 = __shfl_down_sync(0xffffffffu, a0, 8), p2 = __shfl_down_sync(0xffffffffu, a0, 16),
              p3 = __shfl_down_sync(0xffffffffu, a0, 24);
  a0 = __fadd_rn(__fadd_rn(__fadd_rn(a0, p1), p2), p3);
  float total = 0.f;
  for (int i = 8 * V; i < n; ++i) total = __fadd_rn(total, x(i));
#pragma unroll
  for (int l = 0; l < 8; ++l) total = __fadd_rn(total, __shfl_sync(0xffffffffu, a0, l));
  return total;
}

// s_bins[B], s_w[B-1] in; s_cdf[B] scratch.  Writes n_samples values through `emit(j, value)`.
template <class Emit>
__device__ __forceinline__ void sample_pdf_row(const float* s_bins, const float* s_w, float* s_cdf, int B,
                                               const float* __restrict__ u_row, int n_samples, int lane,
                                               Emit emit) {
  const float total = torch_row_sum(s_w, B - 1, lane);                                        // :198-199
  for (int i = lane; i < B - 1; i += 32) s_cdf[i + 1] = __fdiv_rn(__fadd_rn(s_w[i], 1e-5f), total);   // pdf (:199)
  __syncwarp();
  if (lane == 0) {                                  // cumsum (:200-201) as CPU torch: a float64 running sum, each prefix
    double c = 0.0;                                 // rounded to float32
    s_cdf[0] = 0.0f;
    for (int i = 1; i < B; ++i) { c = __dadd_rn(c, (double)s_cdf[i]); s_cdf[i] = __double2float_rn(c); }
  }
  __syncwarp();
  for (int j = lane; j < n_samples; j += 32) {
    const float u = u_row[j];
    int lo = 0, hi = B;                               // first index with cdf > u  (right=True, :223)
    while (lo < hi) { int mid = (lo + hi) >> 1; if (s_cdf[mid] > u) hi = mid; else lo = mid + 1; }
    const int below = max(0, lo - 1), above = min(B - 1, lo);                                 // :224-225
    const float c0 = s_cdf[below], c1 = s_cdf[above], b0 = s_bins[below], b1 = s_bins[above];
    float denom = __fsub_rn(c1, c0);
    if (denom < 1e-5f) denom = 1.0f;                                                          // :235
    const float t = __fdiv_rn(__fsub_rn(u, c0), denom);                                       // :236
    emit(j, __fadd_rn(b0, __fmul_rn(t, __fsub_rn(b1, b0))));                                  // :237
  }
  __syncwarp();
}

__global__ void sample_pdf_kernel(const float* __restrict__ bins, const float* __restrict__ weights,
                                  const float* __restrict__ u, long long u_row_stride, long long N, int B,
                                  int n_samples, float* __restrict__ samples) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  long long n = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (n >= N) return;
  float* s_bins = smem + (size_t)wib * 3 * B;
  float* s_w = s_bins + B;
  float* s_cdf = s_w + B;
  for (int i = lane; i < B; i += 32) s_bins[i] = bins[n * B + i];
  for (int i = lane; i < B - 1; i += 32) s_w[i] = weights[n * (B - 1) + i];
  __syncwarp();
  float* o = samples + n * n_samples;
  sample_pdf_row(s_bins, s_w, s_cdf, B, u + n * u_row_stride, n_samples, lane,
                 [&](int j, float v) { o[j] = v; });
}

// ---------------------------------------------------------------------------------------------
// hierarchical resampling of render_rays (run_nerf.py:392-396, :412): z_mid, sample_pdf on
// weights[1:-1], sort(cat[z, z_samples]), std(z_samples).  One warp per ray.
// ---------------------------------------------------------------------------------------------
__global__ void fine_z_kernel(const float* __restrict__ z_vals, const float* __restrict__ weights,
                              const float* __restrict__ u, long long u_row_stride, long long N, int S,
                              int n_imp, int P /*pow2 >= S+n_imp*/, float* __restrict__ z_fine,
                              float* __restrict__ z_samples_out, float* __restrict__ z_std) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  long long n = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (n >= N) return;
  const int B = S - 1;                                // bins = z_mid [S-1], weights[1:-1] = [S-2]
  float* s_bins = smem + (size_t)wib * (3 * S + P);
  float* s_w = s_bins + S;
  float* s_cdf = s_w + S;
  float* s_all = s_cdf + S;                           // [P] merged z
  for (int i = lane; i < S; i += 32) s_all[i] = z_vals[n * S + i];
  __syncwarp();
  for (int i = lane; i < B; i += 32) s_bins[i] = __fmul_rn(0.5f, __fadd_rn(s_all[i + 1], s_all[i]));   // :392
  for (int i = lane; i < S - 2; i += 32) s_w[i] = weights[n * S + i + 1];                               // :393
  for (int i = S + n_imp + lane; i < P; i += 32) s_all[i] = __int_as_float(0x7f800000);                  // +inf pad
  __syncwarp();
  float* o = s_all + S;
  sample_pdf_row(s_bins, s_w, s_cdf, B, u + n * u_row_stride, n_imp, lane, [&](int j, float v) { o[j] = v; });
  // z_std = std(z_samples, unbiased=False) (:412): CPU torch accumulates in float64 and rounds the result; two-pass float64
  if (z_std) {
    double sum = 0.0;
    for (int j = lane; j < n_imp; j += 32) sum = __dadd_rn(sum, (double)o[j]);
    const double mean = __ddiv_rn(warp_sum_f64(sum), (double)n_imp);
    double var = 0.0;
    for (int j = lane; j < n_imp; j += 32) { const double d = __dsub_rn((double)o[j], mean); var = __dadd_rn(var, __dmul_rn(d, d)); }
    var = __ddiv_rn(warp_sum_f64(var), (double)n_imp);
    if (lane == 0) z_std[n] = __double2float_rn(__dsqrt_rn(var));
  }
  if (z_samples_out) for (int j = lane; j < n_imp; j += 32) z_samples_out[n * n_imp + j] = o[j];
  __syncwarp();
  // sort(cat[z_vals, z_samples]) (:396) by ranking: z_vals is already ascending, so
  //   rank(z_i) = i + #{samples < z_i}            rank(s_j) = #{z <= s_j} + #{s_k < s_j, or == with k < j}
  // (ties resolved z-before-sample and by index: a permutation, like any sort)
  const int SF = S + n_imp;
  float* zout = z_fine + n * SF;
  // the samples are themselves ascending whenever u is (always for det = True: the inverse CDF is monotone);
  // then #{s_k < s_j or tied with k < j} = j and #{samples < z_i} is a lower bound: two binary searches
  // instead of S * n_imp comparisons.  Same permutation as the general path below.
  bool sorted = true;
  for (int j = lane; j + 1 < n_imp; j += 32) sorted = sorted && (o[j] <= o[j + 1]);
  sorted = __all_sync(0xffffffffu, sorted);
  if (sorted) {
    for (int i = lane; i < S; i += 32) {
      const float zi = s_all[i];
      int lo = 0, hi = n_imp;                           // first index with sample >= z_i
      while (lo < hi) { int mid = (lo + hi) >> 1; if (o[mid] < zi) lo = mid + 1; else hi = mid; }
      zout[i + lo] = zi;
    }
    for (int j = lane; j < n_imp; j += 32) {
      const float sj = o[j];
      int lo = 0, hi = S;                               // #{z <= s_j}: first index with z > s_j
      while (lo < hi) { int mid = (lo + hi) >> 1; if (s_all[mid] > sj) hi = mid; else lo = mid + 1; }
      zout[lo + j] = sj;
    }
    return;
  }
  for (int i = lane; i < S; i += 32) {
    const float zi = s_all[i];
    int cnt = 0;
    for (int k = 0; k < n_imp; ++k) cnt += (o[k] < zi) ? 1 : 0;
    zout[i + cnt] = zi;
  }
  for (int j = lane; j < n_imp; j += 32) {
    const float sj = o[j];
    int lo = 0, hi = S;                               // #{z <= s_j}: first index with z > s_j
    while (lo < hi) { int mid = (lo + hi) >> 1; if (s_all[mid] > sj) hi = mid; else lo = mid + 1; }
    int cnt = lo;
    for (int k = 0; k < n_imp; ++k) { const float sk = o[k]; cnt += (sk < sj || (sk == sj && k < j)) ? 1 : 0; }
    zout[cnt] = sj;
  }
}

}  // namespace nb
