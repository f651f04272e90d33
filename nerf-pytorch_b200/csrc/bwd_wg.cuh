// bwd_wg.cuh -- tensor-core backward of one network pass (row a11: loss.backward() through run_nerf.py:381-386 /
// :397-403, i.e. autograd's backward of NeRF.forward run_nerf_helpers.py:96-119 and raw2outputs run_nerf.py:262-305).
//
// Inputs: the per-tile records the training-mode forward left (train_common.cuh: fp16 activation images + ReLU sign
// masks), its raw [N,S,4] output, and dL/drgb_map.  Everything below works on 128-row tiles in the forward's own tile
// order, with activation gradients as loss-scaled fp16 (one power-of-two scale per pass taken from max |dL/drgb_map|,
// saturating conversions) and fp32 accumulation:
//
//   raw2outputs_bwd_kernel (small_kernels.cuh)  dL/draw per sample                       (SURVEY App. E)
//   dhv_seed_heads_kernel  d_hv = relu'(hv) * (d_rgb W_rgb) as tile images + rgb_linear's weight / bias gradient (:114)
//   dA_seed_output_kernel  (no view directions) dA_{D-1} = relu'(a_{D-1}) * (d_raw W_out[:4]) as tile images + output_linear's
//                        weight / bias gradient (:117); the chain below then starts at dA_{D-1}
//   dgrad_wg_kernel      the chain  d_hv -> d_feat -> dA_{D-1} -> ... -> dA_0  as wgmma passes with TRANSPOSED weight chunks
//                        streamed through the forward's weight ring; the epilogue applies the ReLU mask (and the alpha_linear
//                        rank-1 term), writes the next A operand in place and copies it to the gradient record.  Activation
//                        gradients never leave the SM between layers.
//   wgrad_wg_kernel      dW_l += dA_l^T H_{l-1}: both operands MN-major straight from the images (no re-layout), the
//                        CTAs are partitioned over 128-row blocks of the layers' dW so that each holds ONE block in registers
//                        across all of its tiles and writes it once; bias gradients are the column sums of the dA tiles
//                        while they sit in shared memory.
//   wgrad_reduce_kernel  sums the per-CTA partial dW, bias sums and head gradients in CTA order, un-scales, adds into the
//                        gradient tensors (alpha_linear's gradient is computed by the wgrad kernel's MMA warpgroups from the
//                        tiles it streams anyway)
//   dhv_ray_sum_kernel   the per-ray row sums of d_hv, each ray's rows in order
//   views_enc_wgrad_kernel  views_linears[0].weight[:, W:] from the per-ray sums and gamma(viewdir)
//   views_feat_wgrad_kernel views_linears[0].weight[:, :W] = (d_hv^T h_{D-1}) W_feat^T + db_v b_feat^T (feature_linear's output is never stored)
//
// The weight gradient is layer-major because a layer's dW (256 x 256 fp32) is a whole register file: it cannot share a
// kernel with the tile-major dgrad chain.  It streams the images once: 2 x 64 KB per tile-layer at 64 MAC/B -- HBM-bound.
//
// No kernel here adds floats atomically: every sum over rows that several blocks share is written as fp32 partials (one row
// per block, CTA or warp quarter) and added up by a reduction in a fixed order, so that a pass's gradients are the same bits
// on every run (for one tile plan, i.e. one N, S, network and SM count), whatever the scheduling.
#pragma once
#include "fused_tc.cuh"
#include "fused_wg.cuh"
#include "train_common.cuh"

namespace nb {

// ---------------------------------------------------------------------------------------------------------------
// backward weight stream: step 0 = views_linears[0].weight[:, :W]^T (K = W/2: 4 chunks), step 1 = feature_linear^T,
// step j >= 2 = pts_linears[D+1-j].weight[:, h columns]^T (8 chunks each); every chunk is [N = 256 x K = 32] fp16 in the
// forward's SWIZZLE_64B K-major image (pack_weights).  A net without view directions has no steps 0 and 1: its stream
// starts at step 2.
// ---------------------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ int bwd_step_units(int j) { return j == 0 ? 4 : 8; }
static inline int bwd_stream_chunks(int D, int use_viewdirs) { return use_viewdirs ? 4 + 8 * D : 8 * (D - 1); }
// first dgrad step: 0 (d_hv seed -> d_feat -> ...) with view directions, 2 (dA_{D-1} seed) without
__host__ __device__ __forceinline__ int bwd_first_step(int use_viewdirs) { return use_viewdirs ? 0 : 2; }

// ---------------------------------------------------------------------------------------------------------------
// max |g| over n floats -> *out (bit pattern; non-negative floats order like unsigned ints).  *out zeroed by the caller.
// ---------------------------------------------------------------------------------------------------------------
__global__ void absmax_kernel(const float* __restrict__ g, long long n, unsigned int* __restrict__ out) {
  float m = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = fabsf(g[i]);
    m = (v > m || v != v) ? v : m;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const float t = __shfl_xor_sync(0xffffffffu, m, o); m = (t > m || t != t) ? t : m; }
  if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));
}

// gamma(viewdir) per ray (run_nerf.py:44-46 re-encodes it per sample): out [N, ICV]
__global__ void encv_kernel(const float* __restrict__ dirs, int stride, long long N, int ICV, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * ICV) return;
  const long long n = i / ICV;
  const int c = (int)(i - n * ICV);
  const float* d = dirs + n * stride;
  float v;
  if (c < 3) v = d[c];
  else { const int f = (c - 3) / 6, q = (c - 3) % 6; const float a = __fmul_rn(d[q % 3], exp2f((float)f)); v = (q < 3) ? sinf(a) : cosf(a); }
  out[i] = v;
}

// {hi, lo} of a split activation gradient: hi = satfinite(x), lo = satfinite(x - hi) (x - hi exact in fp32 unless hi saturated)
__device__ __forceinline__ void split_sat_f16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
  hi = ptx::cvt_sat_f16x2(a, b);
  const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  lo = ptx::cvt_sat_f16x2(a - hf.x, b - hf.y);
}

// ---------------------------------------------------------------------------------------------------------------
// rgb_linear's backward (run_nerf_helpers.py:114), both halves in one sweep over the rows:
//   seed of the dgrad chain: d_hv[row][c] = scale * (hv[row][c] > 0) * sum_j d_rgb[row][j] W_rgb[j][c]   (c < 128), written as the
//     first 32 KB of every tile's gradient record (rows beyond the CTA's range: zeros -- dgrad and wgrad rely on that);
//   weight / bias gradient: block b's sums over its rows of d_rgb[row][j] hv[row][c] and d_rgb[row][j] (fp32) go to its partial row
//     part[b][SEED_HEADS_PART] = (dW_rgb[3][128], db_rgb[3]); wgrad_reduce_kernel adds the rows in block order
// One warp per row, lane = four columns: a row is 256 contiguous bytes of hv in and of d_hv out (two 128-byte lines each).
// ---------------------------------------------------------------------------------------------------------------
constexpr int SEED_HEADS_PART = 388;      // floats per block: 384 weights + 3 biases (+1: 16-byte rows)
struct SeedParams {
  const float* d_raw; const uint8_t* mask; const uint8_t* act; uint8_t* grad; const float* rgb_w; const unsigned int* amax;
  long long N; int S, rays_per_cta, nst_plan, D;
  uint32_t rec_mask, rec_act, rec_grad; long long n_tiles;
  float* part;
};

// SPLIT (dhv_seed_heads_split_kernel): hv is read as hi + lo (the lo record rec_split_lo above), d_hv is written as
// hi = satfinite(x) and lo = satfinite(x - hi) (the lo gradient record rec_grad_split_lo above); the sums take hv = hi + lo.
template <bool SPLIT>
__device__ __forceinline__ void dhv_seed_heads_body(const SeedParams& p, float (&s_acc)[8][12 * 32 + 3]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = lane * 4, ch = lane >> 4, wsel = (lane >> 3) & 1, bit0 = c & 31;
  const float scale = loss_scale_from_absmax(__uint_as_float(*p.amax));
  float wr[4], wg[4], wb[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { wr[i] = p.rgb_w[c + i] * scale; wg[i] = p.rgb_w[128 + c + i] * scale; wb[i] = p.rgb_w[256 + c + i] * scale; }
  float a[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) a[i] = 0.f;
  float b0 = 0.f, b1 = 0.f, b2 = 0.f;
  for (long long t = blockIdx.x; t < p.n_tiles; t += gridDim.x) {
    const int cta = (int)(t / (2 * p.nst_plan)), st = (int)((t >> 1) % p.nst_plan), X = (int)(t & 1);
    if (st >= plan_cta_nst(p.N, p.S, p.rays_per_cta, cta)) continue;          // never read (the CTA has no rows there)
    const int nrows = plan_cta_rows(p.N, p.S, p.rays_per_cta, cta);
    const int lr0 = st * 256 + X * 128;
    const long long row_begin = (long long)cta * p.rays_per_cta * p.S;
    const int nv = (nrows - lr0 < 128) ? nrows - lr0 : 128;                   // (<= 0: past the CTA's rows -> a tile of zeros)
    const uint8_t* hv = p.act + (size_t)t * p.rec_act + rec_act_hv(p.D);
    const uint8_t* mrec = p.mask + (size_t)t * p.rec_mask + (uint32_t)p.D * 4096u + (uint32_t)ch * 1024u + (uint32_t)wsel * 4u;
    uint8_t* const g = p.grad + (size_t)t * p.rec_grad;
    // warp w takes rows 16 w .. 16 w + 15: their dL/draw rows come in as ONE coalesced load (lane i < 16 holds row i's float4 and
    // hands it out by shuffle), which leaves the registers for all 16 hv / mask loads to be in flight at once (load-latency bound)
    const int rbase = warp * 16;
    float4 dmine = make_float4(0.f, 0.f, 0.f, 0.f);
    if (lane < 16 && rbase + lane < nv) dmine = reinterpret_cast<const float4*>(p.d_raw)[row_begin + lr0 + rbase + lane];
    uint2 hw[16], lw[SPLIT ? 16 : 1];
    uint32_t mw[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const int r = rbase + k;
      hw[k] = make_uint2(0u, 0u); mw[k] = 0u;
      if constexpr (SPLIT) lw[k] = make_uint2(0u, 0u);
      if (r < nv) {
        hw[k] = *reinterpret_cast<const uint2*>(hv + img_off(r, c, 128));
        if constexpr (SPLIT) lw[k] = *reinterpret_cast<const uint2*>(hv + rec_split_lo(p.D) + img_off(r, c, 128));
        mw[k] = *reinterpret_cast<const uint32_t*>(mrec + (uint32_t)r * 8u);
      }
    }
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const int r = rbase + k;
      const float dx = __shfl_sync(0xffffffffu, dmine.x, k), dy = __shfl_sync(0xffffffffu, dmine.y, k), dz = __shfl_sync(0xffffffffu, dmine.z, k);
      uint2 out = make_uint2(0u, 0u), out_lo = make_uint2(0u, 0u);
      if (r < nv) {
        const __half2 h01 = *reinterpret_cast<const __half2*>(&hw[k].x), h23 = *reinterpret_cast<const __half2*>(&hw[k].y);
        float h[4] = {__low2float(h01), __high2float(h01), __low2float(h23), __high2float(h23)};
        if constexpr (SPLIT) {
          const __half2 l01 = *reinterpret_cast<const __half2*>(&lw[k].x), l23 = *reinterpret_cast<const __half2*>(&lw[k].y);
          h[0] += __low2float(l01); h[1] += __high2float(l01); h[2] += __low2float(l23); h[3] += __high2float(l23);
        }
        float x[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          a[i] = fmaf(dx, h[i], a[i]); a[4 + i] = fmaf(dy, h[i], a[4 + i]); a[8 + i] = fmaf(dz, h[i], a[8 + i]);
          x[i] = mask_apply(mw[k], bit0 + i, fmaf(dx, wr[i], fmaf(dy, wg[i], dz * wb[i])));
        }
        b0 += dx; b1 += dy; b2 += dz;
        if constexpr (SPLIT) {
          split_sat_f16x2(x[0], x[1], out.x, out_lo.x);
          split_sat_f16x2(x[2], x[3], out.y, out_lo.y);
        } else {
        out = make_uint2(ptx::cvt_sat_f16x2(x[0], x[1]), ptx::cvt_sat_f16x2(x[2], x[3]));
        }
      }
      *reinterpret_cast<uint2*>(g + img_off(r, c, 128)) = out;
      if constexpr (SPLIT) *reinterpret_cast<uint2*>(g + rec_grad_split_lo(p.D) + img_off(r, c, 128)) = out_lo;
    }
  }
#pragma unroll
  for (int i = 0; i < 12; ++i) s_acc[warp][i * 32 + lane] = a[i];
  if (lane == 0) { s_acc[warp][384] = b0; s_acc[warp][385] = b1; s_acc[warp][386] = b2; }
  __syncthreads();
  for (int i = threadIdx.x; i < 387; i += 256) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) v += s_acc[w][i];
    int o = i;                                          // i = (j * 4 + k) * 32 + lane  ->  weight[j][lane * 4 + k]
    if (i < 384) { const int j = i / 128, k = (i / 32) & 3, ln = i & 31; o = j * 128 + ln * 4 + k; }
    p.part[(size_t)blockIdx.x * SEED_HEADS_PART + o] = v;
  }
}

__global__ void __launch_bounds__(256, 3) dhv_seed_heads_kernel(const SeedParams p) {
  __shared__ float s_acc[8][12 * 32 + 3];
  dhv_seed_heads_body<false>(p, s_acc);
}
// precision TC_SPLIT: the split records (rec_act / rec_grad = the strides of the hi + lo records)
__global__ void __launch_bounds__(256, 1) dhv_seed_heads_split_kernel(const SeedParams p) {
  __shared__ float s_acc[8][12 * 32 + 3];
  dhv_seed_heads_body<true>(p, s_acc);
}

// ---------------------------------------------------------------------------------------------------------------
// output_linear's backward (run_nerf_helpers.py:117: a net without view directions), both halves in one sweep over the rows:
//   seed of the dgrad chain: dA_{D-1}[row][c] = (pre_{D-1}[row][c] > 0) * sum_{k<4} (scale d_raw[row][k]) W_out[k][c], written as
//     the step-1 image of every tile's gradient record -- where the view-direction chain leaves dA_{D-1} too, so that dgrad and
//     wgrad read one layout (rows beyond the CTA's range: zeros, they rely on that);
//   weight / bias gradient: block b's sums over its rows of d_raw[row][k] h_{D-1}[row][c] and d_raw[row][k] (k < 4, fp32) go to its
//     partial row part[b][SEED_OUT_PART] = (dW_out[4][256], db_out[4]); wgrad_reduce_kernel adds the rows in block order (rows >= 4
//     of a 5-output head never reach the loss (run_nerf.py:187) and keep their zero gradient)
// One warp per row, lane = eight columns: a row is 512 contiguous bytes of h_{D-1} in and of dA_{D-1} out.
// ---------------------------------------------------------------------------------------------------------------
constexpr int SEED_OUT_PART = 1028;       // floats per block: 1024 weights + 4 biases
struct SeedOutParams {
  const float* d_raw; const uint8_t* mask; const uint8_t* act; uint8_t* grad; const float* out_w; const unsigned int* amax;
  long long N; int S, rays_per_cta, nst_plan, D;
  uint32_t rec_mask, rec_act, rec_grad; long long n_tiles;
  float* part;
};
constexpr int SEED_OUT_BATCH = 4;         // rows of a warp whose loads are in flight together

// SPLIT (dA_seed_output_split_kernel): h_{D-1} read as hi + lo, dA_{D-1} written as hi and lo images (as dhv_seed_heads_body)
template <bool SPLIT>
__device__ __forceinline__ void dA_seed_output_body(const SeedOutParams& p, float (&s_acc)[8][32 * 32 + 4]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = lane * 8, word = (lane >> 4) * 4 + ((lane >> 2) & 3), bit0 = 8 * (lane & 3);
  const float scale = loss_scale_from_absmax(__uint_as_float(*p.amax));
  float wk[4][8], a[4][8], b[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int i = 0; i < 8; ++i) { wk[k][i] = p.out_w[256 * k + c + i] * scale; a[k][i] = 0.f; }
  for (long long t = blockIdx.x; t < p.n_tiles; t += gridDim.x) {
    const int cta = (int)(t / (2 * p.nst_plan)), st = (int)((t >> 1) % p.nst_plan), X = (int)(t & 1);
    if (st >= plan_cta_nst(p.N, p.S, p.rays_per_cta, cta)) continue;          // never read (the CTA has no rows there)
    const int nrows = plan_cta_rows(p.N, p.S, p.rays_per_cta, cta);
    const int lr0 = st * 256 + X * 128;
    const long long row_begin = (long long)cta * p.rays_per_cta * p.S;
    const int nv = (nrows - lr0 < 128) ? nrows - lr0 : 128;                   // (<= 0: past the CTA's rows -> a tile of zeros)
    const uint8_t* h = p.act + (size_t)t * p.rec_act + rec_act_h(p.D - 1);
    // mask word of this lane's columns: layer D-1, half ch = c >> 7, word (c >> 5) & 3 of the row's uint4
    const uint8_t* mrec = p.mask + (size_t)t * p.rec_mask + (uint32_t)(p.D - 1) * 4096u + (uint32_t)(word >> 2) * 2048u + (uint32_t)(word & 3) * 4u;
    uint8_t* const g = p.grad + (size_t)t * p.rec_grad + rec_grad_step(1);
    // warp w takes rows 16 w .. 16 w + 15; their dL/draw rows come in as one coalesced load (lane i < 16 holds row i's float4)
    const int rbase = warp * 16;
    float4 dmine = make_float4(0.f, 0.f, 0.f, 0.f);
    if (lane < 16 && rbase + lane < nv) dmine = reinterpret_cast<const float4*>(p.d_raw)[row_begin + lr0 + rbase + lane];
    for (int r8 = 0; r8 < 16; r8 += SEED_OUT_BATCH) {
      uint4 hw[SEED_OUT_BATCH], lw[SPLIT ? SEED_OUT_BATCH : 1];
      uint32_t mw[SEED_OUT_BATCH];
#pragma unroll
      for (int k = 0; k < SEED_OUT_BATCH; ++k) {
        const int r = rbase + r8 + k;
        hw[k] = make_uint4(0u, 0u, 0u, 0u); mw[k] = 0u;
        if constexpr (SPLIT) lw[k] = make_uint4(0u, 0u, 0u, 0u);
        if (r < nv) {
          hw[k] = *reinterpret_cast<const uint4*>(h + img_off(r, c, 256));
          if constexpr (SPLIT) lw[k] = *reinterpret_cast<const uint4*>(h + rec_split_lo(p.D) + img_off(r, c, 256));
          mw[k] = *reinterpret_cast<const uint32_t*>(mrec + (uint32_t)r * 16u);
        }
      }
#pragma unroll
      for (int k = 0; k < SEED_OUT_BATCH; ++k) {
        const int r = rbase + r8 + k;
        const float d[4] = {__shfl_sync(0xffffffffu, dmine.x, r8 + k), __shfl_sync(0xffffffffu, dmine.y, r8 + k),
                            __shfl_sync(0xffffffffu, dmine.z, r8 + k), __shfl_sync(0xffffffffu, dmine.w, r8 + k)};
        uint4 out = make_uint4(0u, 0u, 0u, 0u), out_lo = make_uint4(0u, 0u, 0u, 0u);
        if (r < nv) {
          const uint32_t hu[4] = {hw[k].x, hw[k].y, hw[k].z, hw[k].w};
          float x[8];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const __half2 hh = *reinterpret_cast<const __half2*>(&hu[q]);
            float hv2[2] = {__low2float(hh), __high2float(hh)};
            if constexpr (SPLIT) {
              const uint32_t lu[4] = {lw[k].x, lw[k].y, lw[k].z, lw[k].w};
              const __half2 ll = *reinterpret_cast<const __half2*>(&lu[q]);
              hv2[0] += __low2float(ll); hv2[1] += __high2float(ll);
            }
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int i = 2 * q + e;
#pragma unroll
              for (int kk = 0; kk < 4; ++kk) a[kk][i] = fmaf(d[kk], hv2[e], a[kk][i]);
              x[i] = mask_apply(mw[k], bit0 + i, fmaf(d[0], wk[0][i], fmaf(d[1], wk[1][i], fmaf(d[2], wk[2][i], d[3] * wk[3][i]))));
            }
          }
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) b[kk] += d[kk];
          if constexpr (SPLIT) {
            split_sat_f16x2(x[0], x[1], out.x, out_lo.x); split_sat_f16x2(x[2], x[3], out.y, out_lo.y);
            split_sat_f16x2(x[4], x[5], out.z, out_lo.z); split_sat_f16x2(x[6], x[7], out.w, out_lo.w);
          } else {
          out = make_uint4(ptx::cvt_sat_f16x2(x[0], x[1]), ptx::cvt_sat_f16x2(x[2], x[3]), ptx::cvt_sat_f16x2(x[4], x[5]), ptx::cvt_sat_f16x2(x[6], x[7]));
          }
        }
        *reinterpret_cast<uint4*>(g + img_off(r, c, 256)) = out;
        if constexpr (SPLIT) *reinterpret_cast<uint4*>(g + rec_grad_split_lo(p.D) + img_off(r, c, 256)) = out_lo;
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int i = 0; i < 8; ++i) s_acc[warp][(8 * k + i) * 32 + lane] = a[k][i];
  if (lane == 0) { s_acc[warp][1024] = b[0]; s_acc[warp][1025] = b[1]; s_acc[warp][1026] = b[2]; s_acc[warp][1027] = b[3]; }
  __syncthreads();
  for (int i = threadIdx.x; i < 1028; i += 256) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) v += s_acc[w][i];
    int o = i;                                          // i = (k * 8 + e) * 32 + lane  ->  weight[k][lane * 8 + e]
    if (i < 1024) { const int k = i >> 8, e = (i >> 5) & 7, ln = i & 31; o = k * 256 + ln * 8 + e; }
    p.part[(size_t)blockIdx.x * SEED_OUT_PART + o] = v;
  }
}

__global__ void __launch_bounds__(256, 2) dA_seed_output_kernel(const SeedOutParams p) {
  __shared__ float s_acc[8][32 * 32 + 4];
  dA_seed_output_body<false>(p, s_acc);
}
// precision TC_SPLIT: the split records (rec_act / rec_grad = the strides of the hi + lo records)
__global__ void __launch_bounds__(256, 1) dA_seed_output_split_kernel(const SeedOutParams p) {
  __shared__ float s_acc[8][32 * 32 + 4];
  dA_seed_output_body<true>(p, s_acc);
}

// ---------------------------------------------------------------------------------------------------------------
// dgrad chain -- the warpgroup roles, weight ring and operand layout of march_wg_kernel (fused_wg.cuh), with the backward
// weight stream (transposed chunks) and the gradient record: each MMA warpgroup loads its 64 rows of the tile's d_hv seed
// (16 KB, one bulk copy), then runs steps j = 0..D: step 0 = d_hv W_v[:, :W] -> d_feat, step j >= 1 = the previous step's
// output times the transposed weights of the layer above -> (+ d_sigma alpha_linear.weight at j = 1) -> ReLU mask of pts layer
// D - j from the forward's sign bits -> saturating fp16, in place as the next step's A operand and, byte for byte, the
// warpgroup's half of the step's image in the gradient record (one 32 KB bulk store).
// Without view directions (first_step = 2) the seed is dA_{D-1} itself (dA_seed_output_kernel, the step-1 image): each MMA
// warpgroup loads its 32 KB half straight into its A operand and the chain runs steps 2..D; d_raw and alpha_w are not read.
// ---------------------------------------------------------------------------------------------------------------
struct DgradParams {
  const uint8_t* mask; uint8_t* grad; const float* d_raw; const unsigned int* amax; const float* alpha_w;
  const uint8_t* chunks;                    // backward weight stream (pack_weights), starting at step first_step
  long long N; int S, rays_per_cta, nst_plan, D;
  uint32_t rec_mask, rec_grad;
  int vc0, vc1;                             // forward CTAs [vc0, vc1): this launch's CTA b serves vc0 + b, vc0 + b + gridDim, ...
  int first_step;                           // 0: d_hv seed (view directions), 2: dA_{D-1} seed (output_linear head)
};

// The split chain (dgrad_split_kernel, precision TC_SPLIT): every operand is a hi and a lo fp16 image.  Its map: the hi A operands
// at 0, alpha_linear.weight and the barriers in the 16 KB above them, the lo A operands SPLIT_LO above the hi ones (the split
// forward's offset), then a ring of DS_NST stages of [N = 256 x K = 16] hi | lo columns (the split packed image's backward stream).
// The seed goes straight into the A operands (hi and lo), as the fp16 chain's dA_{D-1} seed does.
constexpr int DS_NST = 5;
constexpr uint32_t DS_ALPHA = 65536;                             // alpha_linear.weight, 1 KB
constexpr uint32_t DS_BARS = DS_ALPHA + 1024;                    // full, empty [DS_NST], seed [2]
constexpr uint32_t DS_WRING = SPLIT_LO + 65536;                  // 147456
constexpr uint32_t DS_ALLOC = DS_WRING + DS_NST * TC_STAGE_BYTES;   // 229376
static_assert(DS_BARS + 16 * DS_NST + 16 <= SPLIT_LO && DS_ALLOC <= 227 * 1024, "the split chain's shared-memory map");

// layer of the forward whose (transposed) weights step j multiplies by: the view layer, feature_linear, pts_linears[D + 1 - j]
__host__ __device__ __forceinline__ int bwd_step_layer(int j, int D) { return j == 0 ? D + 1 : D + 1 - j; }

template <bool SPLIT>
__device__ __forceinline__ void dgrad_chain(const DgradParams& p, const float* wscale) {
  constexpr int NST = SPLIT ? DS_NST : TC_NST;
  uint8_t* smem = tc_smem;
  const uint32_t sb = ptx::smem_u32(smem);
  if ((sb & 1023u) != 0) __trap();
  float* s_alpha = reinterpret_cast<float*>(smem + (SPLIT ? DS_ALPHA : SM_HEADS));
  const int D = p.D, NS = D + 1, j0 = p.first_step;
  const uint32_t bars = sb + (SPLIT ? DS_BARS : SM_BARS);
  RingN<NST> rg{bars, bars + 8 * NST, 0, 0};
  const uint32_t bar_seed = bars + 16 * NST;                     // [2]: one per MMA warpgroup
  if (j0 == 0)
    for (int i = threadIdx.x; i < 256; i += TC_THREADS) s_alpha[i] = p.alpha_w[i];
  if (threadIdx.x == 0) {
    for (int i = 0; i < NST; ++i) { ptx::mbar_init(rg.full + 8 * i, 1); ptx::mbar_init(rg.empty + 8 * i, 256); }
    ptx::mbar_init(bar_seed, 1); ptx::mbar_init(bar_seed + 8, 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();

  if (threadIdx.x < 128) {
    // =========================== producer: the backward chunk stream, once per tile ===========================
    ptx::setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      for (int vc = p.vc0 + (int)blockIdx.x; vc < p.vc1; vc += (int)gridDim.x)
        for (int tile = 0, nt = 2 * plan_cta_nst(p.N, p.S, p.rays_per_cta, vc); tile < nt; ++tile) {
          const uint8_t* src = p.chunks;
          for (int j = j0; j < NS; ++j)
            for (int u = 0; u < bwd_step_units(j) * (SPLIT ? 2 : 1); ++u) {
              ptx::mbar_wait(rg.empty + 8 * rg.stage, rg.phase ^ 1);
              ptx::mbar_arrive_expect_tx(rg.full + 8 * rg.stage, TC_STAGE_BYTES);
              ptx::bulk_g2s(sb + (SPLIT ? DS_WRING : SM_WRING) + rg.stage * TC_STAGE_BYTES, src, TC_STAGE_BYTES, rg.full + 8 * rg.stage);
              src += TC_STAGE_BYTES;
              rg.advance();
            }
        }
    }
    return;
  }

  // =========================== MMA warpgroups ===========================
  ptx::setmaxnreg_inc<232>();
  const int w = (threadIdx.x >> 7) - 1, t = threadIdx.x & 127, wq = t >> 5, lane = t & 31;
  const int q4 = lane & 3;
  const int r0 = 16 * wq + (lane >> 2), r1 = r0 + 8;
  const uint32_t act = sb + SM_ACT + (uint32_t)w * 32768u, seed = SPLIT ? act : sb + SM_ENC + (uint32_t)w * 16384u;
  const uint32_t ring = sb + (SPLIT ? DS_WRING : SM_WRING);
  const uint32_t glo = SPLIT ? rec_grad_split_lo(D) : 0u;       // the lo gradient record above the hi one
  const float scale = loss_scale_from_absmax(__uint_as_float(*p.amax));
  const uint64_t l2_first = ptx::l2_policy_evict_first();
  auto wg_sync = [&]() { ptx::named_bar_sync(1 + w, 128); };
  const uint32_t ro0 = (uint32_t)((r0 >> 3) * 1024 + (r0 & 7) * 128 + 4 * q4), ro1 = (uint32_t)((r1 >> 3) * 1024 + (r1 & 7) * 128 + 4 * q4);
  auto pair_addr = [&](uint32_t ro, int r, int j) { return act + ro + (uint32_t)(j >> 3) * 8192u + (uint32_t)(((j & 7) ^ (r & 7)) << 4); };
  uint32_t sph = 0;
  float acc[128];
  Phases none;
  for (int vc = p.vc0 + (int)blockIdx.x; vc < p.vc1; vc += (int)gridDim.x) {
    const int nrows = plan_cta_rows(p.N, p.S, p.rays_per_cta, vc);
    const int nt = 2 * plan_cta_nst(p.N, p.S, p.rays_per_cta, vc);
    const long long row_begin = (long long)vc * p.rays_per_cta * p.S;
    for (int tile = 0; tile < nt; ++tile) {
      const int st = tile >> 1, X = tile & 1;
      const long long tid = ((long long)vc * p.nst_plan + st) * 2 + X;
      const uint8_t* const mrec = p.mask + (size_t)tid * p.rec_mask;
      uint8_t* const grec = p.grad + (size_t)tid * p.rec_grad;
      const int lrb = st * TC_ST + X * TC_TILE + 64 * w;
      // the warpgroup's 64 rows of the seed (the MMAs of the previous tile's step 0 have read the buffer); a dA_{D-1} seed goes
      // to the A operand, once the previous tile's last record copy has read it.  SPLIT: both seeds go to the A operands (hi, lo).
      if (t == 0) {
        if constexpr (SPLIT) {
          const uint32_t sbytes = j0 == 0 ? 16384u : 32768u;
          const uint8_t* src = grec + (j0 == 0 ? (uint32_t)w * 16384u : rec_grad_step(1) + (uint32_t)w * 32768u);
          ptx::bulk_wait_read0();
          ptx::mbar_arrive_expect_tx(bar_seed + 8 * w, 2 * sbytes);
          ptx::bulk_g2s(act, src, sbytes, bar_seed + 8 * w);
          ptx::bulk_g2s(act + SPLIT_LO, src + glo, sbytes, bar_seed + 8 * w);
        } else if (j0 == 0) {
          ptx::mbar_arrive_expect_tx(bar_seed + 8 * w, 16384u);
          ptx::bulk_g2s(seed, grec + (uint32_t)w * 16384u, 16384u, bar_seed + 8 * w);
        } else {
          ptx::bulk_wait_read0();
          ptx::mbar_arrive_expect_tx(bar_seed + 8 * w, 32768u);
          ptx::bulk_g2s(act, grec + rec_grad_step(1) + (uint32_t)w * 32768u, 32768u, bar_seed + 8 * w);
        }
      }
      float dsig[2] = {0.f, 0.f};
      if (j0 == 0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int lr = lrb + (h ? r1 : r0);
          dsig[h] = lr < nrows ? p.d_raw[(row_begin + lr) * 4 + 3] * scale : 0.f;
        }
      }
      ptx::mbar_wait(bar_seed + 8 * w, sph);
      sph ^= 1;
      for (int j = j0; j < NS; ++j) {
        // ReLU mask of this step's output (the pre-activation of pts layer D - j), fetched before the MMAs
        uint4 mk[2][2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int ch = 0; ch < 2; ++ch)
            mk[h][ch] = (j >= 1) ? *reinterpret_cast<const uint4*>(mrec + (uint32_t)(D - j) * 4096u + (uint32_t)ch * 2048u + (uint32_t)(64 * w + (h ? r1 : r0)) * 16u)
                                 : make_uint4(0u, 0u, 0u, 0u);
        const uint32_t abase = (j == 0) ? seed : act;
        auto a_of = [&](int c) { return desc_act(abase + (uint32_t)(c >> 1) * 8192u + (uint32_t)(c & 1) * 64u); };
        float isc = 1.0f;
        if constexpr (SPLIT) {
          mma_layer_split(acc, rg, ring, 2 * bwd_step_units(j), true, a_of, none);
          isc = 1.0f / wscale[bwd_step_layer(j, D)];
        } else {
          mma_layer(acc, rg, ring, bwd_step_units(j), true, a_of);
        }
        if (t == 0) ptx::bulk_wait_read0();                     // the previous step's record copy has read the operand
        wg_sync();
#pragma unroll
        for (int jj = 0; jj < 32; ++jj) {
          const int c = 8 * jj + 2 * q4;
          float x[2][2] = {{acc[4 * jj], acc[4 * jj + 1]}, {acc[4 * jj + 2], acc[4 * jj + 3]}};
          if constexpr (SPLIT) {                                // undo the weights' power-of-two scale (exact)
#pragma unroll
            for (int h = 0; h < 2; ++h) { x[h][0] *= isc; x[h][1] *= isc; }
          }
          if (j == 1) {                                         // + d_sigma * alpha_linear.weight (run_nerf_helpers.py:106)
            const float2 a = *reinterpret_cast<const float2*>(s_alpha + c);
#pragma unroll
            for (int h = 0; h < 2; ++h) { x[h][0] = fmaf(dsig[h], a.x, x[h][0]); x[h][1] = fmaf(dsig[h], a.y, x[h][1]); }
          }
          if (j >= 1) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const uint4 m4 = mk[h][c >> 7];
              const int wi = (c >> 5) & 3;
              const uint32_t m = wi == 0 ? m4.x : wi == 1 ? m4.y : wi == 2 ? m4.z : m4.w;
              x[h][0] = mask_apply(m, c & 31, x[h][0]);
              x[h][1] = mask_apply(m, (c & 31) + 1, x[h][1]);
            }
          }
          if constexpr (SPLIT) {
            uint32_t h0, l0, h1, l1;
            split_sat_f16x2(x[0][0], x[0][1], h0, l0);
            split_sat_f16x2(x[1][0], x[1][1], h1, l1);
            ptx::st_shared_b32(pair_addr(ro0, r0, jj), h0);
            ptx::st_shared_b32(pair_addr(ro1, r1, jj), h1);
            ptx::st_shared_b32(pair_addr(ro0, r0, jj) + SPLIT_LO, l0);
            ptx::st_shared_b32(pair_addr(ro1, r1, jj) + SPLIT_LO, l1);
          } else {
          ptx::st_shared_b32(pair_addr(ro0, r0, jj), ptx::cvt_sat_f16x2(x[0][0], x[0][1]));
          ptx::st_shared_b32(pair_addr(ro1, r1, jj), ptx::cvt_sat_f16x2(x[1][0], x[1][1]));
          }
        }
        ptx::fence_proxy_async_smem();
        wg_sync();
        if (t == 0) {
          ptx::bulk_s2g_hint(grec + rec_grad_step(j) + (uint32_t)w * 32768u, act, 32768u, l2_first);
          if constexpr (SPLIT) ptx::bulk_s2g_hint(grec + glo + rec_grad_step(j) + (uint32_t)w * 32768u, act + SPLIT_LO, 32768u, l2_first);
          ptx::bulk_commit();
        }
      }
    }
  }
  if (t == 0) ptx::bulk_wait_all();
}

__global__ void __launch_bounds__(TC_THREADS, 1) dgrad_wg_kernel(const DgradParams p) {
  dgrad_chain<false>(p, nullptr);
}
// precision TC_SPLIT: the chain on split operands (three MMAs per K = 16 step), p.chunks = the split training image's backward
// stream, wscale = its per-layer weight scales, p.rec_grad = the stride of the hi + lo gradient records
__global__ void __launch_bounds__(TC_THREADS, 1) dgrad_split_kernel(const DgradParams p, const float* __restrict__ wscale) {
  dgrad_chain<true>(p, wscale);
}

// ---------------------------------------------------------------------------------------------------------------
// wgrad: layer-major.  Job = one weight block dW[128 x Nc] = sum over tiles of A_t^T B_t, A = 128 columns (from m0) of a
// gradient image, B = an activation image (Nc columns); a contiguous range of CTAs serves a job, CTA g of G takes the job's
// tiles g, g + G, ...  Stage = one 64-row half tile of A's 128 columns and of B (one contiguous piece each in the record).
// Warpgroup 0: one producer thread.  Warpgroups 1, 2: wgmma with both operands MN-major straight from the images, each on 64
// of the block's rows (dW rows = A columns), the accumulator in registers for the whole launch; while the MMAs of a stage
// run, the same threads form the bias gradient (column sums of A) and alpha_linear's gradient from the stage in shared memory.
// ---------------------------------------------------------------------------------------------------------------
constexpr int WG2_THREADS = 384, WG2_MAX_STAGES = 6, WG2_MAX_JOBS = 24;
constexpr uint32_t WG2_RING = 196608,                  // ring: 4 stages of a 128 + 256 column job
                   WG2_BARS = WG2_RING, WG2_TOTAL = WG2_BARS + 256;

struct WgradJob {
  uint32_t a_off, b_off;        // image offsets inside the gradient / activation record
  int a_cols, m0;               // columns of the A image (128 | 256); first A column of this block (0 | 128)
  int Nc;                       // columns of B (64 | 128 | 256)
  int cta0, ncta;               // CTA range serving this job
  long long part_off;           // float offset of this job's partial blocks [ncta][128][Nc]
  long long db_off;             // -1, or float offset of the scaled column sums of A (bias gradient) [ncta][4][128]
  long long alpha_off;          // -1, or (B = h_{D-1}) float offset of alpha_linear's partials: [ncta][2][256] weight
                                // (sum_rows d_sigma[row] B[row][c]), then [ncta][2] bias (sum_rows d_sigma[row])
};
struct WgradParams {
  const uint8_t* act; const uint8_t* grad; uint32_t rec_act, rec_grad;
  long long N; int S, rays_per_cta, nst_plan; long long n_tiles;
  float* partial; const float* d_raw; int njobs;
  long long t0, t1;             // tiles [t0, t1) of the plan (a launch may cover part of a pass; the reduction adds up)
  WgradJob jobs[WG2_MAX_JOBS];
};

__device__ __forceinline__ bool plan_tile_valid(const WgradParams& p, long long t) {
  const int cta = (int)(t / (2 * p.nst_plan)), st = (int)((t >> 1) % p.nst_plan);
  return st < plan_cta_nst(p.N, p.S, p.rays_per_cta, cta);
}

// byte offset of (row r < 64, even column c < 64) inside one 8 KB K-block of a half image
__device__ __forceinline__ uint32_t kblock_off(int r, int c) {
  return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + (((c >> 3) ^ (r & 7)) << 4) + (c & 7) * 2);
}

template <int NC>
__device__ __forceinline__ void wgrad_consumer(const WgradParams& p, const WgradJob& job, int g, int G, uint32_t sb, uint32_t stride,
                                               uint32_t nstg, uint32_t bar_full, uint32_t bar_empty) {
  constexpr int R = NC / 2;
  const int w = (threadIdx.x >> 7) - 1, t = threadIdx.x & 127, wq = t >> 5, lane = t & 31;
  const int cp = t & 31;                                  // column pair of the bias sums: A columns m0 + 64 w + 2 cp, rows 16 wq ..
  const int cp2 = t & 63, rh = t >> 6;                    // alpha_linear: B columns 128 w + 2 cp2, rows 32 rh ..
  float acc[R];
#pragma unroll
  for (int i = 0; i < R; ++i) acc[i] = 0.f;
  float s0 = 0.f, s1 = 0.f, a0 = 0.f, a1 = 0.f, bsum = 0.f;
  uint32_t s = 0, ph = 0;
  bool any = false;
  for (long long tt = p.t0 + g; tt < p.t1; tt += G) {
    if (!plan_tile_valid(p, tt)) continue;
    const int cta = (int)(tt / (2 * p.nst_plan)), st = (int)((tt >> 1) % p.nst_plan), X = (int)(tt & 1);
    const int nrows = plan_cta_rows(p.N, p.S, p.rays_per_cta, cta);
    const long long row_begin = (long long)cta * p.rays_per_cta * p.S;
    for (int h = 0; h < 2; ++h) {
      const int lr0 = st * 256 + X * 128 + h * 64;
      const uint32_t xb = sb + s * stride, yb = xb + 16384u;
      float dsv = 0.f;
      if (job.alpha_off >= 0) { const int lr = lr0 + 32 * rh + lane; dsv = lr < nrows ? p.d_raw[(row_begin + lr) * 4 + 3] : 0.f; }
      ptx::mbar_wait(bar_full + 8 * s, ph);
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t ad = ptx::gmma_desc(xb + (uint32_t)w * 8192u + k * 2048, 8192, 1024, ptx::GMMA_SW128);
        const uint64_t bd = ptx::gmma_desc(yb + k * 2048, 8192, 1024, ptx::GMMA_SW128);
        const uint32_t accum = (any || k > 0) ? 1u : 0u;
        if constexpr (NC == 256) ptx::wgmma_m64n256k16<1, 1>(acc, ad, bd, accum);
        else if constexpr (NC == 128) ptx::wgmma_m64n128k16<1, 1>(acc, ad, bd, accum);
        else ptx::wgmma_m64n64k16<1, 1>(acc, ad, bd, accum);
      }
      ptx::wgmma_commit();
      any = true;
      // while the MMAs run: column sums of this warpgroup's 64 A columns (bias gradient)
      if (job.db_off >= 0) {
        const uint32_t abase = xb + (uint32_t)w * 8192u;
        for (int i = 0; i < 16; ++i) {
          const uint32_t v = ptx::ld_shared_b32(abase + kblock_off(16 * wq + i, 2 * cp));
          const __half2 hh = *reinterpret_cast<const __half2*>(&v);
          s0 += __low2float(hh); s1 += __high2float(hh);
        }
      }
      if (job.alpha_off >= 0) {                                  // alpha_linear.weight: sum_rows d_sigma[row] h_{D-1}[row][c]
        const int c = 128 * w + 2 * cp2;
        const uint32_t bbase = yb + (uint32_t)(c >> 6) * 8192u;
#pragma unroll 8
        for (int i = 0; i < 32; ++i) {
          const float d = __shfl_sync(0xffffffffu, dsv, i);
          const int r = 32 * rh + i;
          const uint32_t v = ptx::ld_shared_b32(bbase + kblock_off(r, c & 63));
          const __half2 hh = *reinterpret_cast<const __half2*>(&v);
          a0 = fmaf(d, __low2float(hh), a0); a1 = fmaf(d, __high2float(hh), a1);
          bsum += d;
        }
      }
      ptx::wgmma_wait<0>();
      ptx::fence_regs(acc);
      ptx::mbar_arrive(bar_empty + 8 * s);
      if (++s == nstg) { s = 0; ph ^= 1; }
    }
  }
  // every CTA writes all of its partials (zeros when it had no tiles): the reduction reads them all
  if (job.db_off >= 0)
    *reinterpret_cast<float2*>(p.partial + job.db_off + ((size_t)g * 4 + wq) * 128 + 64 * w + 2 * cp) = make_float2(s0, s1);
  if (job.alpha_off >= 0) {
    *reinterpret_cast<float2*>(p.partial + job.alpha_off + ((size_t)g * 2 + rh) * 256 + 128 * w + 2 * cp2) = make_float2(a0, a1);
    if (w == 0 && cp2 == 0) p.partial[job.alpha_off + (size_t)G * 512 + g * 2 + rh] = bsum;
  }
  float* part = p.partial + job.part_off + (size_t)g * 128 * NC;
  const int q4 = lane & 3, rr = 64 * w + 16 * wq + (lane >> 2);
#pragma unroll
  for (int j = 0; j < NC / 8; ++j) {
    const int c = 8 * j + 2 * q4;
    *reinterpret_cast<float2*>(part + (size_t)rr * NC + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
    *reinterpret_cast<float2*>(part + (size_t)(rr + 8) * NC + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
  }
}

__global__ void __launch_bounds__(WG2_THREADS, 1) wgrad_wg_kernel(const WgradParams p) {
  uint8_t* smem = tc_smem;
  const uint32_t sb = ptx::smem_u32(smem);
  if ((sb & 1023u) != 0) __trap();
  int ji = -1;
  for (int i = 0; i < p.njobs; ++i) if ((int)blockIdx.x >= p.jobs[i].cta0 && (int)blockIdx.x < p.jobs[i].cta0 + p.jobs[i].ncta) ji = i;
  if (ji < 0) return;                                   // (uniform per CTA, before any barrier)
  const WgradJob job = p.jobs[ji];
  const int g = (int)blockIdx.x - job.cta0, G = job.ncta;
  const uint32_t bar_full = sb + WG2_BARS, bar_empty = sb + WG2_BARS + 8 * WG2_MAX_STAGES;
  const int ykb = job.Nc >> 6;
  const uint32_t stride = 16384u + (uint32_t)ykb * 8192u;
  // as many stages of this job's size as fit (narrow jobs get more: the bytes in flight per SM set its share of the bus)
  const uint32_t nstg = (WG2_RING / stride < (uint32_t)WG2_MAX_STAGES) ? WG2_RING / stride : (uint32_t)WG2_MAX_STAGES;
  if (threadIdx.x == 0) {
    for (int i = 0; i < WG2_MAX_STAGES; ++i) { ptx::mbar_init(bar_full + 8 * i, 1); ptx::mbar_init(bar_empty + 8 * i, 256); }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x < 128) {
    ptx::setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      uint32_t s = 0, ph = 0;
      for (long long t = p.t0 + g; t < p.t1; t += G) {
        if (!plan_tile_valid(p, t)) continue;
        for (int h = 0; h < 2; ++h) {
          ptx::mbar_wait(bar_empty + 8 * s, ph ^ 1);
          ptx::mbar_arrive_expect_tx(bar_full + 8 * s, stride);
          // 64-row half tile h of each operand: its K-blocks are adjacent in the record -> one contiguous piece per operand
          const uint8_t* xs = p.grad + (size_t)t * p.rec_grad + job.a_off + (size_t)h * (job.a_cols >> 6) * 8192 + (size_t)(job.m0 >> 6) * 8192;
          const uint8_t* ys = p.act + (size_t)t * p.rec_act + job.b_off + (size_t)h * ykb * 8192;
          ptx::bulk_g2s(sb + s * stride, xs, 16384u, bar_full + 8 * s);
          ptx::bulk_g2s(sb + s * stride + 16384u, ys, (uint32_t)ykb * 8192u, bar_full + 8 * s);
          if (++s == nstg) { s = 0; ph ^= 1; }
        }
      }
    }
    return;
  }
  ptx::setmaxnreg_inc<232>();
  if (job.Nc == 256) wgrad_consumer<256>(p, job, g, G, sb, stride, nstg, bar_full, bar_empty);
  else if (job.Nc == 128) wgrad_consumer<128>(p, job, g, G, sb, stride, nstg, bar_full, bar_empty);
  else wgrad_consumer<64>(p, job, g, G, sb, stride, nstg, bar_full, bar_empty);
}

// dst[o][i] += (scaled ? inv_scale : 1) * sum_g partial[g][o][i], g = 0, 1, ... in order   (i < n_valid; dst row stride ldw;
// partial rows g are gstride floats apart).  A dW job has Mc = 128 (one block); the others are bias and head gradients.
struct ReduceJob { long long part_off, gstride; int ncta, Mc, Nc, n_valid, ldw, scaled; float* dst; };
constexpr int WG2_MAX_REDUCE = 56;        // dW blocks, their bias sums, alpha_linear and the seed kernels' heads
struct ReduceParams { const float* partial; const unsigned int* amax; int njobs; ReduceJob jobs[WG2_MAX_REDUCE]; };

__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const ReduceParams p) {
  const ReduceJob j = p.jobs[blockIdx.y];
  const int idx = blockIdx.x * 256 + threadIdx.x;
  if (idx >= j.Mc * j.Nc) return;
  const int o = idx / j.Nc, i = idx - o * j.Nc;
  if (i >= j.n_valid) return;
  const float* src = p.partial + j.part_off + idx;
  float s = 0.f;
  for (int g = 0; g < j.ncta; ++g) s += src[(size_t)g * j.gstride];
  const float inv = j.scaled ? 1.0f / loss_scale_from_absmax(__uint_as_float(*p.amax)) : 1.0f;
  j.dst[(size_t)o * j.ldw + i] += s * inv;
}

// ---------------------------------------------------------------------------------------------------------------
// the view columns of views_linears[0] (alpha_linear rides along in the wgrad kernel, whose tiles already hold its operands;
// rgb_linear's gradient comes from dhv_seed_heads_kernel)
// ---------------------------------------------------------------------------------------------------------------
// dsum[ray][c] = inv_scale * sum over the ray's rows, in order, of d_hv[row][c]: one warp per ray, lane = four columns, walking the
// ray's rows through the tile plan in the d_hv seed images (offset 0 of each gradient record).  A ray's rows may span tiles and
// super-tiles but never CTAs (whole rays per CTA).
constexpr int DSUM_BATCH = 8;             // rows of a warp whose loads are in flight together
// SPLIT (dhv_ray_sum_split_kernel): each row is hi + lo (the lo record `lo` bytes above), added in fp32 before the running sum
template <bool SPLIT>
__device__ __forceinline__ void dhv_ray_sum_body(const uint8_t* __restrict__ grad, uint32_t rec_grad, uint32_t lo, long long N, int S,
                                                 int rays_per_cta, int nst_plan, const unsigned int* __restrict__ amax, float* __restrict__ dsum) {
  const long long n = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (n >= N) return;
  const int c = (threadIdx.x & 31) * 4;
  const int cta = (int)(n / rays_per_cta), lr0 = (int)(n - (long long)cta * rays_per_cta) * S;
  const uint8_t* rec = grad + (size_t)cta * nst_plan * 2 * rec_grad;      // the CTA's tiles: local row lr is in tile lr >> 7
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  for (int k0 = 0; k0 < S; k0 += DSUM_BATCH) {
    uint2 v[DSUM_BATCH], vl[SPLIT ? DSUM_BATCH : 1];
#pragma unroll
    for (int k = 0; k < DSUM_BATCH; ++k) {
      const int lr = lr0 + k0 + k;
      v[k] = (k0 + k < S) ? *reinterpret_cast<const uint2*>(rec + (size_t)(lr >> 7) * rec_grad + img_off(lr & 127, c, 128)) : make_uint2(0u, 0u);
      if constexpr (SPLIT)
        vl[k] = (k0 + k < S) ? *reinterpret_cast<const uint2*>(rec + (size_t)(lr >> 7) * rec_grad + lo + img_off(lr & 127, c, 128)) : make_uint2(0u, 0u);
    }
#pragma unroll
    for (int k = 0; k < DSUM_BATCH; ++k) {
      if (k0 + k < S) {
        const __half2 h01 = *reinterpret_cast<const __half2*>(&v[k].x), h23 = *reinterpret_cast<const __half2*>(&v[k].y);
        if constexpr (SPLIT) {
          const __half2 l01 = *reinterpret_cast<const __half2*>(&vl[k].x), l23 = *reinterpret_cast<const __half2*>(&vl[k].y);
          s[0] += __low2float(h01) + __low2float(l01); s[1] += __high2float(h01) + __high2float(l01);
          s[2] += __low2float(h23) + __low2float(l23); s[3] += __high2float(h23) + __high2float(l23);
        } else {
        s[0] += __low2float(h01); s[1] += __high2float(h01); s[2] += __low2float(h23); s[3] += __high2float(h23);
        }
      }
    }
  }
  const float inv = 1.0f / loss_scale_from_absmax(__uint_as_float(*amax));
  *reinterpret_cast<float4*>(dsum + n * 128 + c) = make_float4(s[0] * inv, s[1] * inv, s[2] * inv, s[3] * inv);
}
__global__ void __launch_bounds__(256) dhv_ray_sum_kernel(const uint8_t* __restrict__ grad, uint32_t rec_grad, long long N, int S,
                                                        int rays_per_cta, int nst_plan, const unsigned int* __restrict__ amax,
                                                        float* __restrict__ dsum) {
  dhv_ray_sum_body<false>(grad, rec_grad, 0u, N, S, rays_per_cta, nst_plan, amax, dsum);
}
// precision TC_SPLIT: rec_grad = the stride of the hi + lo gradient records, lo = the lo record's offset
__global__ void __launch_bounds__(256) dhv_ray_sum_split_kernel(const uint8_t* __restrict__ grad, uint32_t rec_grad, uint32_t lo, long long N, int S,
                                                              int rays_per_cta, int nst_plan, const unsigned int* __restrict__ amax,
                                                              float* __restrict__ dsum) {
  dhv_ray_sum_body<true>(grad, rec_grad, lo, N, S, rays_per_cta, nst_plan, amax, dsum);
}

// Block (e, b) sums over the rays [b R, (b + 1) R): part[b][c][e] = sum dsum[ray][c] * gamma(viewdir_ray)[e] for e < ICV (the view
// columns of views_linears[0].weight, run_nerf_helpers.py:108-110), and part[b][ICV][c] = sum dsum[ray][c] (this pass's bias
// gradient of views_linears[0], for views_feat_wgrad_kernel).  gridDim.y is set by the SM count, not by N; wgrad_reduce_kernel
// adds the blocks' rows in order.  part: [gridDim.y][(ICV + 1) * 128]
__global__ void __launch_bounds__(128) views_enc_wgrad_kernel(const float* __restrict__ dsum, const float* __restrict__ encv, long long N, int ICV,
                                                            long long R, float* __restrict__ part) {
  const int e = blockIdx.x, c = threadIdx.x;
  const long long n0 = (long long)blockIdx.y * R, n1 = (n0 + R < N) ? n0 + R : N;
  float* row = part + (size_t)blockIdx.y * (ICV + 1) * 128;
  float s = 0.f;
  if (e < ICV) {
    for (long long n = n0; n < n1; ++n) s = fmaf(dsum[n * 128 + c], encv[n * ICV + e], s);
    row[c * ICV + e] = s;
  } else {
    for (long long n = n0; n < n1; ++n) s += dsum[n * 128 + c];
    row[ICV * 128 + c] = s;
  }
}

// views_linears[0].weight[v][f] (f < W) += sum_k G[v][k] W_feat[f][k] + dbv[v] b_feat[f], with G = d_hv^T h_{D-1} (the views job of
// the wgrad kernel, already reduced and un-scaled): the feature layer has no activation, so
//   d_hv^T feat = d_hv^T (h_{D-1} W_feat^T + 1 b_feat^T) = G W_feat^T + (sum_rows d_hv) b_feat^T
// and feature_linear's output never has to be stored (run_nerf_helpers.py:107-110).  grid = 128 (v), block = 256 (f).
__global__ void __launch_bounds__(256) views_feat_wgrad_kernel(const float* __restrict__ G, const float* __restrict__ dbv, const float* __restrict__ feat_w,
                                                             const float* __restrict__ feat_b, float* __restrict__ views_w, int ld) {
  __shared__ float s_g[256];
  const int v = blockIdx.x, f = threadIdx.x;
  s_g[f] = G[v * 256 + f];
  __syncthreads();
  const float4* w4 = reinterpret_cast<const float4*>(feat_w + (size_t)f * 256);
  float acc = dbv[v] * feat_b[f];
#pragma unroll 8
  for (int k4 = 0; k4 < 64; ++k4) {
    const float4 w = w4[k4];
    acc = fmaf(s_g[4 * k4], w.x, acc); acc = fmaf(s_g[4 * k4 + 1], w.y, acc); acc = fmaf(s_g[4 * k4 + 2], w.z, acc); acc = fmaf(s_g[4 * k4 + 3], w.w, acc);
  }
  views_w[(size_t)v * ld + f] += acc;
}

}  // namespace nb
