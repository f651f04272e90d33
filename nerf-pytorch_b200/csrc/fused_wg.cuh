// fused_wg.cuh -- the fused network pass on Hopper warpgroup MMA (wgmma): pts = o + d*z -> positional encoding ->
// 8x256 MLP (+ heads) -> alpha compositing, run_nerf.py:381-386 / :397-403 (run_network :37-51, Embedder.embed
// run_nerf_helpers.py:36-45, NeRF.forward :96-119, raw2outputs run_nerf.py:262-305).
//
// One CTA per SM walks its whole rays in 128-row tiles (the tile plan of train_common.cuh).  Warpgroup 0 is the producer: one
// thread streams the packed weight chunks ([N = 256 x K = 32] fp16, 16 KB, SWIZZLE_64B K-major) through a ring of TC_NST
// stages with cp.async.bulk.  Warpgroups 1 and 2 each own 64 rows of the tile: they encode their rows into the layer-0 A
// operand, issue the layer's wgmma.m64n256k16 chain (A = their activation K-blocks, B = the ring stage; the accumulator
// starts at the fp32 bias) and run the epilogue in registers -- ReLU, fp16, stored in place as the next layer's A operand,
// the heads as fp32 FMA chains on the pre-rounding activations, the per-ray view bias in the view layer -- then composite
// the tile's rows with segmented warp scans and a carry handed warp to warp.  A ring stage is released when both MMA
// warpgroups' wgmma groups that read it have completed (every consumer thread arrives on the stage's empty barrier).
//
// Training mode (EMIT): each warpgroup's A operand is byte for byte its half of the tile image in the record, so after a layer's
// epilogue one thread copies the 32 KB (encodings 8 KB, view layer 16 KB) to the record with cp.async.bulk shared -> global,
// and waits for the copy to finish reading before the next epilogue overwrites the operand.  The sign bits of the
// pre-activations go out as 8-byte stores (mask record, train_common.cuh).
#pragma once
#include "fused_tc.cuh"
#include "train_common.cuh"

namespace nb {

// training-mode save buffers of one pass (train_common.cuh)
struct TrainSaveDev { uint8_t* act; uint8_t* mask; int nst_plan; uint32_t rec_act, rec_mask; };

// byte offset of (row r < 64, even column c) in a warpgroup's A operand: K-blocks of 64 columns x 64 rows, SWIZZLE_128B
__device__ __forceinline__ uint32_t half_off(int r, int c) {
  return (uint32_t)((c >> 6) * 8192 + (r >> 3) * 1024 + (r & 7) * 128 + ((((c & 63) >> 3) ^ (r & 7)) << 4) + (c & 7) * 2);
}

// K-major operand descriptors: activations (SWIZZLE_128B, 8-row groups of 1 KB) and weight chunks (SWIZZLE_64B, 512 B)
__device__ __forceinline__ uint64_t desc_act(uint32_t addr) { return ptx::gmma_desc(addr, 16, 1024, ptx::GMMA_SW128); }
__device__ __forceinline__ uint64_t desc_w(uint32_t addr) { return ptx::gmma_desc(addr, 16, 512, ptx::GMMA_SW64); }

// Phase counters of an experiments build (-DNERF_B200_PHASE_PROBE, tools/forward_phase_probe.py): thread 0 of each MMA
// warpgroup adds the clock64 time it spends in each phase to g_fwd_phase[slot][CTA][warpgroup][phase], slot = the launch
// count modulo PH_SLOTS (coarse, fine).  PH_FULL: waits on a ring stage's full barrier; PH_GAP: from the end of a layer's
// MMAs (wgmma_wait<0>) to the next layer's first full-barrier wait, inside a tile; PH_SAMPLER / PH_COMPOSITOR: from the
// tile's start to its first layer / from its last layer's epilogue to its end; PH_TOTAL: the warpgroup's whole run.  The
// product build compiles all of it to nothing.
enum { PH_FULL, PH_GAP, PH_SAMPLER, PH_COMPOSITOR, PH_TOTAL, PH_N };
#ifdef NERF_B200_PHASE_PROBE
constexpr int PH_SLOTS = 2, PH_MAX_CTAS = 1024;
__device__ unsigned long long g_fwd_phase[PH_SLOTS][PH_MAX_CTAS][2][PH_N];
__device__ int g_fwd_phase_slot;
struct Phases {
  long long acc[PH_N] = {0, 0, 0, 0, 0}, t0 = 0, tb = 0;
  __device__ __forceinline__ void begin() { tb = clock64(); }
  __device__ __forceinline__ void start() { t0 = clock64(); }
  __device__ __forceinline__ void stop(int k) { acc[k] += clock64() - t0; }
  __device__ __forceinline__ void wait_full(uint32_t bar, uint32_t parity) {
    const long long a = clock64();
    ptx::mbar_wait(bar, parity);
    acc[PH_FULL] += clock64() - a;
  }
  __device__ __forceinline__ void flush(int w, int t) {
    acc[PH_TOTAL] = clock64() - tb;
    if (t == 0 && blockIdx.x < PH_MAX_CTAS)
      for (int k = 0; k < PH_N; ++k) atomicAdd(&g_fwd_phase[g_fwd_phase_slot][blockIdx.x][w][k], (unsigned long long)acc[k]);
  }
};
#else
struct Phases {
  __device__ __forceinline__ void begin() {}
  __device__ __forceinline__ void start() {}
  __device__ __forceinline__ void stop(int) {}
  __device__ __forceinline__ void wait_full(uint32_t bar, uint32_t parity) { ptx::mbar_wait(bar, parity); }
  __device__ __forceinline__ void flush(int, int) {}
};
#endif

// Weight ring shared by the producer and both MMA warpgroups: every party walks the same chunk sequence.
template <int NST>
struct RingN {
  uint32_t full, empty, stage, phase;
  __device__ __forceinline__ void advance() { if (++stage == NST) { stage = 0; phase ^= 1; } }
};
using Ring = RingN<TC_NST>;

// One K = 32 chunk into a 64 x N accumulator (two K = 16 instructions); `acc0` = 0 overwrites the accumulator
template <int R>
__device__ __forceinline__ void mma_chunk(float (&acc)[R], uint64_t ad, uint64_t bd, uint32_t acc0) {
  if constexpr (R == 128) {
    ptx::wgmma_m64n256k16<0, 0>(acc, ad, bd, acc0);
    ptx::wgmma_m64n256k16<0, 0>(acc, ad + 2, bd + 2, 1u);
  } else {
    ptx::wgmma_m64n128k16<0, 0>(acc, ad, bd, acc0);
    ptx::wgmma_m64n128k16<0, 0>(acc, ad + 2, bd + 2, 1u);
  }
}

// All chunks of one layer: `a_of(c)` gives chunk c's A descriptor.  The previous chunk's stage is released as soon as the
// wgmma group of the next one is in flight; on return the accumulator is complete.
template <int R, typename RG, typename AOf>
__device__ __forceinline__ void mma_layer(float (&acc)[R], RG& rg, uint32_t ring_base, int nch, bool from_zero, AOf a_of, Phases& ph) {
  ptx::wgmma_fence();
  int pending = -1;
  for (int c = 0; c < nch; ++c) {
    const uint32_t s = rg.stage;
    ph.wait_full(rg.full + 8 * s, rg.phase);
    mma_chunk(acc, a_of(c), desc_w(ring_base + s * TC_STAGE_BYTES), (from_zero && c == 0) ? 0u : 1u);
    ptx::wgmma_commit();
    if (pending >= 0) { ptx::wgmma_wait<1>(); ptx::mbar_arrive(rg.empty + 8 * pending); }
    pending = (int)s;
    rg.advance();
  }
  ptx::wgmma_wait<0>();
  ptx::fence_regs(acc);
  if (pending >= 0) ptx::mbar_arrive(rg.empty + 8 * pending);
}
template <int R, typename AOf>
__device__ __forceinline__ void mma_layer(float (&acc)[R], Ring& rg, uint32_t ring_base, int nch, bool from_zero, AOf a_of) {
  Phases none;
  mma_layer(acc, rg, ring_base, nch, from_zero, a_of, none);
}

// The split forward's layer: stage c holds K = 16 columns of chunk c >> 1 (hi | lo), `a_of(c >> 1)` gives the chunk's hi A
// descriptor and the lo image is SPLIT_LO above it.  Three MMAs per stage into the one accumulator: hi_a hi_b, hi_a lo_b, lo_a hi_b.
template <int R, typename RG, typename AOf>
__device__ __forceinline__ void mma_layer_split(float (&acc)[R], RG& rg, uint32_t ring_base, int nst, bool from_zero, AOf a_of, Phases& ph) {
  ptx::wgmma_fence();
  int pending = -1;
  for (int c = 0; c < nst; ++c) {
    const uint32_t s = rg.stage;
    ph.wait_full(rg.full + 8 * s, rg.phase);
    const uint64_t ah = a_of(c >> 1) + (uint64_t)(2 * (c & 1)), al = ah + (SPLIT_LO >> 4);
    const uint64_t bd = desc_w(ring_base + s * TC_STAGE_BYTES);
    if constexpr (R == 128) {
      ptx::wgmma_m64n256k16<0, 0>(acc, ah, bd, (from_zero && c == 0) ? 0u : 1u);
      ptx::wgmma_m64n256k16<0, 0>(acc, ah, bd + 2, 1u);
      ptx::wgmma_m64n256k16<0, 0>(acc, al, bd, 1u);
    } else {
      ptx::wgmma_m64n128k16<0, 0>(acc, ah, bd, (from_zero && c == 0) ? 0u : 1u);
      ptx::wgmma_m64n128k16<0, 0>(acc, ah, bd + 2, 1u);
      ptx::wgmma_m64n128k16<0, 0>(acc, al, bd, 1u);
    }
    ptx::wgmma_commit();
    if (pending >= 0) { ptx::wgmma_wait<1>(); ptx::mbar_arrive(rg.empty + 8 * pending); }
    pending = (int)s;
    rg.advance();
  }
  ptx::wgmma_wait<0>();
  ptx::fence_regs(acc);
  if (pending >= 0) ptx::mbar_arrive(rg.empty + 8 * pending);
}

// {hi, lo} fp16 pairs of (a, b): hi = fp16(x), lo = fp16(x - hi), x - hi exact in fp32
__device__ __forceinline__ void split_f16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
  hi = ptx::cvt_f16x2(a, b);
  const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  lo = ptx::cvt_f16x2(a - hf.x, b - hf.y);
}

// OR of a value over the four lanes that share an accumulator row
__device__ __forceinline__ uint32_t quad_or(uint32_t v) {
  v |= __shfl_xor_sync(0xffffffffu, v, 1);
  return v | __shfl_xor_sync(0xffffffffu, v, 2);
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// The density grid of density_wg_kernel / density_split_kernel: column n = i * ny + j of the pass is the "ray" of the nz points
// (xs[i], ys[j], zs[k]), k = 0 .. nz - 1 (p.S = nz), and row m = n * nz + k of the pass is sigma's C-order index.
struct DensityGrid { const float* xs; const float* ys; const float* zs; int ny; float* sigma; };

// The pass of march_wg_kernel (SPLIT false) and march_split_kernel / march_split_train_kernel (SPLIT true).  SPLIT: every MMA
// operand is a hi and a lo fp16 image (the split map of fused_tc.cuh), each weight chunk streams as two ring stages, the weights
// are scaled by wscale[l] (a power of two: the accumulator starts at bias * wscale[l] and is scaled back exactly after the MMAs).
// EMIT && SPLIT: a tile's record is the hi record followed by the lo record (rec_split_lo), and every image goes out twice: the
// hi operand and the lo operand SPLIT_LO above it.
// DENSITY (never EMIT): the points come from the axes of `grid`, only the pts layers stream and run, and the sigma head
// (alpha_linear, or row 3 of output_linear without view directions) goes straight out as one fp32 per row: no view layers,
// view bias, raw rows or compositing.  The head is the same code in the same order as the other modes, so sigma is bit for bit
// raw[..., 3] of the pts mode on the same points.
template <bool EMIT, bool SPLIT, bool DENSITY = false>
__device__ __forceinline__ void march_pass(const MarchParams p, const TrainSaveDev sv, const float* wscale, const DensityGrid grid = {}) {
  static_assert(!(EMIT && DENSITY), "the density pass has no training mode");
  constexpr int NST = SPLIT ? SPLIT_NST : FWD_NST;
  constexpr int CPS = SPLIT ? 2 : 1;                              // ring stages per weight chunk
  uint8_t* smem = tc_smem;
  const uint32_t sb = ptx::smem_u32(smem);
  if ((sb & 1023u) != 0) __trap();
  float* s_heads = reinterpret_cast<float*>(smem + FWD_HEADS);
  float* s_bias = reinterpret_cast<float*>(smem + FWD_BIAS);
  const uint32_t a_heads = sb + FWD_HEADS, a_carry = sb + FWD_MISC;
  const int D = p.D, NL = DENSITY ? p.D : p.D + (p.use_viewdirs ? 2 : 0);

  // this CTA's rays / rows; the number of super-tiles is the tile plan's (train_common.cuh: plan_cta_nst)
  const long long ray0 = (long long)blockIdx.x * p.rays_per_cta;
  const int nrows = plan_cta_rows(p.N, p.S, p.rays_per_cta, blockIdx.x);
  const int nst = plan_cta_nst(p.N, p.S, p.rays_per_cta, blockIdx.x);
  const long long row_begin = ray0 * p.S;

  for (int i = threadIdx.x; i < HEADS_FLOATS; i += TC_THREADS) s_heads[i] = p.heads[i];
  for (int i = threadIdx.x; i < (TC_MAXD + 1) * 256; i += TC_THREADS) s_bias[i] = p.bias[i];
  RingN<NST> rg{sb + FWD_BARS, sb + FWD_BARS + 8 * NST, 0, 0};
  if (threadIdx.x == 0) {
    for (int i = 0; i < NST; ++i) { ptx::mbar_init(rg.full + 8 * i, 1); ptx::mbar_init(rg.empty + 8 * i, 256); }
    sts32(a_carry + CARRY_T, 1.0f); sts32(a_carry + CARRY_R, 0.f); sts32(a_carry + CARRY_G, 0.f); sts32(a_carry + CARRY_B, 0.f);
    sts32(a_carry + CARRY_D, 0.f); sts32(a_carry + CARRY_A, 0.f); st_release_shared(a_carry + CARRY_TURN, 0u);
    ptx::fence_mbar_init();
  }
  __syncthreads();

  if (threadIdx.x < 128) {
    // =========================== producer: the chunk stream, once per tile ===========================
    ptx::setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      for (int tile = 0; tile < 2 * nst; ++tile) {
        const uint8_t* src = p.chunks;
        for (int l = 0; l < NL; ++l) {
          const int nch = tc_layer_chunks(l, D, p.skip) * CPS;
          const uint32_t bytes = tc_layer_chunk_bytes(l, D);
          for (int c = 0; c < nch; ++c) {
            ptx::mbar_wait(rg.empty + 8 * rg.stage, rg.phase ^ 1);
            ptx::mbar_arrive_expect_tx(rg.full + 8 * rg.stage, bytes);
            ptx::bulk_g2s(sb + (SPLIT ? SPLIT_WRING : FWD_WRING) + rg.stage * TC_STAGE_BYTES, src, bytes, rg.full + 8 * rg.stage);
            src += bytes;
            rg.advance();
          }
        }
      }
    }
    return;
  }

  // =========================== MMA warpgroups ===========================
  ptx::setmaxnreg_inc<232>();
  const int w = (threadIdx.x >> 7) - 1, t = threadIdx.x & 127, wq = t >> 5, lane = t & 31;
  const int q4 = lane & 3;
  const int r0 = 16 * wq + (lane >> 2), r1 = r0 + 8;              // this thread's two accumulator rows (of the warpgroup's 64)
  const uint32_t act = sb + SM_ACT + (uint32_t)w * 32768u, enc = sb + FWD_ENC + (uint32_t)w * 8192u;
  const uint32_t ring = sb + (SPLIT ? SPLIT_WRING : FWD_WRING);
  const uint64_t l2_first = EMIT ? ptx::l2_policy_evict_first() : 0ull;
  const uint32_t rec_lo = rec_split_lo(D);                       // EMIT && SPLIT: lo record -> its tile's hi record
  auto wg_sync = [&]() { ptx::named_bar_sync(1 + w, 128); };
  // row-dependent parts of the swizzled addresses of this thread's pairs: column pair (8 j + 2 q4) of row r sits at
  // rowoff(r) + (j >> 3) * 8192 + (((j & 7) ^ (r & 7)) << 4) + 4 q4
  const uint32_t ro0 = (uint32_t)((r0 >> 3) * 1024 + (r0 & 7) * 128 + 4 * q4), ro1 = (uint32_t)((r1 >> 3) * 1024 + (r1 & 7) * 128 + 4 * q4);
  auto pair_addr = [&](uint32_t base, uint32_t ro, int r, int j) { return base + ro + (uint32_t)(j >> 3) * 8192u + (uint32_t)(((j & 7) ^ (r & 7)) << 4); };
  // stmatrix row address of this lane: row 16 wq + 8 ((lane >> 3) & 1) + (lane & 7), column group j + (lane >> 4) for even j,
  // whose swizzled 16-byte chunk is (j & 7) ^ sm_key
  const int sm_r = 16 * wq + 8 * ((lane >> 3) & 1) + (lane & 7);
  const uint32_t sm_row = act + act_row_off(sm_r), sm_key = (uint32_t)((lane >> 4) ^ (lane & 7));

  float acc[128];
  Phases ph;
  ph.begin();
  for (int tile = 0; tile < 2 * nst; ++tile) {
    ph.start();
    const int st = tile >> 1, X = tile & 1;
    uint8_t* const arec = EMIT ? sv.act + (size_t)((blockIdx.x * sv.nst_plan + st) * 2 + X) * sv.rec_act : nullptr;
    uint8_t* const mrec = EMIT ? sv.mask + (size_t)((blockIdx.x * sv.nst_plan + st) * 2 + X) * sv.rec_mask : nullptr;
    const int lrb = st * TC_ST + X * TC_TILE + 64 * w;            // row (inside the CTA's range) of the warpgroup's row 0
    long long nray[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int lr = lrb + (h ? r1 : r0);
      const int rl = (lr < nrows ? lr : nrows - 1) / p.S;
      long long n = ray0 + rl;
      nray[h] = n > p.N - 1 ? p.N - 1 : (n < 0 ? 0 : n);
    }

    // ---- sampler: pts = o + d z (run_nerf.py:381) and the positional encoding of the warpgroup's 64 rows ----
    if (EMIT && t == 0) ptx::bulk_wait_read0();                  // the previous tile's copies have read the operands
    wg_sync();
    if (t < 64) {
      const int lr = lrb + t;
      float px = 0.f, py = 0.f, pz = 0.f;
      if (lr < nrows) {
        const long long m = row_begin + lr;
        if constexpr (DENSITY) {
          const long long n = m / p.S;
          px = grid.xs[n / grid.ny]; py = grid.ys[n % grid.ny]; pz = grid.zs[m - n * p.S];
        } else if (p.pts) { px = p.pts[m * 3]; py = p.pts[m * 3 + 1]; pz = p.pts[m * 3 + 2]; }
        else {
          const float* ry = p.rays + (ray0 + lr / p.S) * p.ray_stride;
          const float z = p.z_vals[m];
          px = __fadd_rn(ry[0], __fmul_rn(ry[3], z));
          py = __fadd_rn(ry[1], __fmul_rn(ry[4], z));
          pz = __fadd_rn(ry[2], __fmul_rn(ry[5], z));
        }
      }
      if constexpr (SPLIT) encode_row_store_split(enc + act_row_off(t), enc + SPLIT_LO + act_row_off(t), t, px, py, pz, p.L);
      else encode_row_store(enc + act_row_off(t), t, px, py, pz, p.L);
    }
    ptx::fence_proxy_async_smem();
    wg_sync();
    if (EMIT && t == 0) {
      ptx::bulk_s2g_hint(arec + (uint32_t)w * 8192u, enc, 8192u, l2_first);
      if constexpr (SPLIT) ptx::bulk_s2g_hint(arec + rec_lo + (uint32_t)w * 8192u, enc + SPLIT_LO, 8192u, l2_first);
      ptx::bulk_commit();
    }

    float hp[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};   // head partial sums of this thread's columns, per row
    ph.stop(PH_SAMPLER);
    for (int l = 0; l < NL; ++l) {
      const int nch = tc_layer_chunks(l, D, p.skip);
      const bool skip_layer = (l < D && p.skip >= 0 && l == p.skip + 1);
      auto a_of = [&](int c) -> uint64_t {
        if (l == 0 || (skip_layer && c < 2)) return desc_act(enc + (uint32_t)c * 64u);
        const int k = skip_layer ? c - 2 : c;
        return desc_act(act + (uint32_t)(k >> 1) * 8192u + (uint32_t)(k & 1) * 64u);
      };
      if (l <= D) {
        // ---- pts_linears[l] (ReLU) or feature_linear (no activation): 64 x 256 ----
        const float* bias = s_bias + 256 * l;
        if constexpr (SPLIT) {
          const float sc = wscale[l], isc = 1.0f / sc;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const float2 b = *reinterpret_cast<const float2*>(bias + 8 * j + 2 * q4);
            acc[4 * j] = b.x * sc; acc[4 * j + 1] = b.y * sc; acc[4 * j + 2] = b.x * sc; acc[4 * j + 3] = b.y * sc;
          }
          if (l > 0) ph.stop(PH_GAP);
          mma_layer_split(acc, rg, ring, nch * 2, false, a_of, ph);
#pragma unroll
          for (int i = 0; i < 128; ++i) acc[i] *= isc;
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const float2 b = *reinterpret_cast<const float2*>(bias + 8 * j + 2 * q4);
            acc[4 * j] = b.x; acc[4 * j + 1] = b.y; acc[4 * j + 2] = b.x; acc[4 * j + 3] = b.y;
          }
          if (l > 0) ph.stop(PH_GAP);
          mma_layer(acc, rg, ring, nch, false, a_of, ph);
        }
        ph.start();
        if (EMIT && t == 0) ptx::bulk_wait_read0();
        wg_sync();                                                // the whole warpgroup's MMAs and copies are done with the operand
        const bool last_pts = (l == D - 1);
        if (EMIT && l < D) {
          uint32_t m0[8], m1[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) { m0[i] = 0u; m1[i] = 0u; }
#pragma unroll
          for (int j = 0; j < 32; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int bit = 31 - (8 * (j & 3) + 2 * q4 + e);
              m0[j >> 2] |= (__float_as_uint(acc[4 * j + e]) >> 31) << bit;
              m1[j >> 2] |= (__float_as_uint(acc[4 * j + 2 + e]) >> 31) << bit;
            }
          uint2 v0 = make_uint2(0u, 0u), v1 = make_uint2(0u, 0u);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            m0[i] = quad_or(m0[i]); m1[i] = quad_or(m1[i]);
          }
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (q4 == k) { v0 = make_uint2(m0[2 * k], m0[2 * k + 1]); v1 = make_uint2(m1[2 * k], m1[2 * k + 1]); }
          const uint32_t mo = (uint32_t)l * 4096u + (uint32_t)(q4 >> 1) * 2048u + (uint32_t)(q4 & 1) * 8u;
          *reinterpret_cast<uint2*>(mrec + mo + (uint32_t)(64 * w + r0) * 16u) = v0;
          *reinterpret_cast<uint2*>(mrec + mo + (uint32_t)(64 * w + r1) * 16u) = v1;
        }
        if (last_pts) {
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const int c = 8 * j + 2 * q4;
            const float a0 = fmaxf(acc[4 * j], 0.f), a1 = fmaxf(acc[4 * j + 1], 0.f), b0 = fmaxf(acc[4 * j + 2], 0.f), b1 = fmaxf(acc[4 * j + 3], 0.f);
            if (p.use_viewdirs) {                                 // alpha_linear (run_nerf_helpers.py:106)
              const float2 wa = *reinterpret_cast<const float2*>(s_heads + c);
              hp[0][3] = fmaf(a1, wa.y, fmaf(a0, wa.x, hp[0][3]));
              hp[1][3] = fmaf(b1, wa.y, fmaf(b0, wa.x, hp[1][3]));
            } else {                                              // output_linear (:117); DENSITY: its sigma row only
#pragma unroll
              for (int k = DENSITY ? 3 : 0; k < 4; ++k) {
                const float2 wk = *reinterpret_cast<const float2*>(s_heads + 256 * k + c);
                hp[0][k] = fmaf(a1, wk.y, fmaf(a0, wk.x, hp[0][k]));
                hp[1][k] = fmaf(b1, wk.y, fmaf(b0, wk.x, hp[1][k]));
              }
            }
          }
        }
        // without view directions only the fp32 head above reads h_{D-1}: inference skips the fp16 image, training mode still
        // records it (output_linear's weight gradient reads it, dA_seed_output_kernel in bwd_wg.cuh); the density pass ends there
        if (EMIT || !(last_pts && (DENSITY || !p.use_viewdirs))) {
          const bool relu = l < D;
          // column groups j, j + 1 of the warp's 16 rows as four 8 x 8 matrices (the accumulator fragment is stmatrix's):
          // matrix m = (group j + (m >> 1), rows + 8 (m & 1)); this lane addresses row (lane & 7) of matrix lane >> 3
#pragma unroll
          for (int j = 0; j < 32; j += 2) {
            uint32_t h[4];
            if constexpr (SPLIT) {
              uint32_t lo[4];
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int g = j + e;
                const float x0 = relu ? fmaxf(acc[4 * g], 0.f) : acc[4 * g], x1 = relu ? fmaxf(acc[4 * g + 1], 0.f) : acc[4 * g + 1];
                const float y0 = relu ? fmaxf(acc[4 * g + 2], 0.f) : acc[4 * g + 2], y1 = relu ? fmaxf(acc[4 * g + 3], 0.f) : acc[4 * g + 3];
                split_f16x2(x0, x1, h[2 * e], lo[2 * e]);
                split_f16x2(y0, y1, h[2 * e + 1], lo[2 * e + 1]);
              }
              ptx::stmatrix_x4(sm_row + SPLIT_LO + (uint32_t)(j >> 3) * 8192u + ((uint32_t)((j & 7) ^ sm_key) << 4), lo[0], lo[1], lo[2], lo[3]);
            } else {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int g = j + e;
              h[2 * e] = relu ? ptx::cvt_relu_f16x2(acc[4 * g], acc[4 * g + 1]) : ptx::cvt_f16x2(acc[4 * g], acc[4 * g + 1]);
              h[2 * e + 1] = relu ? ptx::cvt_relu_f16x2(acc[4 * g + 2], acc[4 * g + 3]) : ptx::cvt_f16x2(acc[4 * g + 2], acc[4 * g + 3]);
            }
            }
            ptx::stmatrix_x4(sm_row + (uint32_t)(j >> 3) * 8192u + ((uint32_t)((j & 7) ^ sm_key) << 4), h[0], h[1], h[2], h[3]);
          }
          ptx::fence_proxy_async_smem();
          wg_sync();
          if (EMIT && l < D && t == 0) {
            ptx::bulk_s2g_hint(arec + rec_act_h(l) + (uint32_t)w * 32768u, act, 32768u, l2_first);
            if constexpr (SPLIT) ptx::bulk_s2g_hint(arec + rec_lo + rec_act_h(l) + (uint32_t)w * 32768u, act + SPLIT_LO, 32768u, l2_first);
            ptx::bulk_commit();
          }
        }
      } else {
        // ---- views_linears[0] (N = 128) + per-ray view bias, ReLU, rgb_linear ----
        float* accv = acc;                                        // the first 64 accumulators
        if constexpr (SPLIT) {
          const float isc = 1.0f / wscale[l];
          ph.stop(PH_GAP);
          mma_layer_split(*reinterpret_cast<float(*)[64]>(accv), rg, ring, nch * 2, true, a_of, ph);
#pragma unroll
          for (int i = 0; i < 64; ++i) acc[i] *= isc;
        } else {
          ph.stop(PH_GAP);
          mma_layer(*reinterpret_cast<float(*)[64]>(accv), rg, ring, nch, true, a_of, ph);
        }
        ph.start();
        wg_sync();
        const float* vb0 = p.vb + nray[0] * 128;
        const float* vb1 = p.vb + nray[1] * 128;
        uint32_t m0[4] = {0u, 0u, 0u, 0u}, m1[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int c = 8 * j + 2 * q4;
          const float2 b0 = *reinterpret_cast<const float2*>(vb0 + c), b1 = *reinterpret_cast<const float2*>(vb1 + c);
          const float x0 = acc[4 * j] + b0.x, x1 = acc[4 * j + 1] + b0.y, y0 = acc[4 * j + 2] + b1.x, y1 = acc[4 * j + 3] + b1.y;
          if (EMIT) {
            const int bit = 31 - (8 * (j & 3) + 2 * q4);
            m0[j >> 2] |= ((__float_as_uint(x0) >> 31) << bit) | ((__float_as_uint(x1) >> 31) << (bit - 1));
            m1[j >> 2] |= ((__float_as_uint(y0) >> 31) << bit) | ((__float_as_uint(y1) >> 31) << (bit - 1));
            if constexpr (SPLIT) {
              uint32_t h0, l0, h1, l1;
              split_f16x2(fmaxf(x0, 0.f), fmaxf(x1, 0.f), h0, l0);
              split_f16x2(fmaxf(y0, 0.f), fmaxf(y1, 0.f), h1, l1);
              ptx::st_shared_b32(pair_addr(act, ro0, r0, j), h0);
              ptx::st_shared_b32(pair_addr(act, ro1, r1, j), h1);
              ptx::st_shared_b32(pair_addr(act + SPLIT_LO, ro0, r0, j), l0);
              ptx::st_shared_b32(pair_addr(act + SPLIT_LO, ro1, r1, j), l1);
            } else {
            ptx::st_shared_b32(pair_addr(act, ro0, r0, j), ptx::cvt_relu_f16x2(x0, x1));
            ptx::st_shared_b32(pair_addr(act, ro1, r1, j), ptx::cvt_relu_f16x2(y0, y1));
            }
          }
          const float h00 = fmaxf(x0, 0.f), h01 = fmaxf(x1, 0.f), h10 = fmaxf(y0, 0.f), h11 = fmaxf(y1, 0.f);
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            const float2 wk = *reinterpret_cast<const float2*>(s_heads + 256 + 128 * k + c);
            hp[0][k] = fmaf(h01, wk.y, fmaf(h00, wk.x, hp[0][k]));
            hp[1][k] = fmaf(h11, wk.y, fmaf(h10, wk.x, hp[1][k]));
          }
        }
        if (EMIT) {
#pragma unroll
          for (int i = 0; i < 4; ++i) { m0[i] = quad_or(m0[i]); m1[i] = quad_or(m1[i]); }
          uint32_t v0 = 0u, v1 = 0u;
#pragma unroll
          for (int k = 0; k < 4; ++k) if (q4 == k) { v0 = m0[k]; v1 = m1[k]; }
          const uint32_t mo = (uint32_t)D * 4096u + (uint32_t)(q4 >> 1) * 1024u + (uint32_t)(q4 & 1) * 4u;
          *reinterpret_cast<uint32_t*>(mrec + mo + (uint32_t)(64 * w + r0) * 8u) = v0;
          *reinterpret_cast<uint32_t*>(mrec + mo + (uint32_t)(64 * w + r1) * 8u) = v1;
          ptx::fence_proxy_async_smem();
          wg_sync();
          if (t == 0) {
            ptx::bulk_s2g_hint(arec + rec_act_hv(D) + (uint32_t)w * 16384u, act, 16384u, l2_first);
            if constexpr (SPLIT) ptx::bulk_s2g_hint(arec + rec_lo + rec_act_hv(D) + (uint32_t)w * 16384u, act + SPLIT_LO, 16384u, l2_first);
            ptx::bulk_commit();
          }
        }
      }
    }

    if constexpr (DENSITY) {
      // ---- the sigma head's row sum over the quad (as raw[h][3] below) -> sigma ----
      const float s0 = quad_sum(hp[0][3]), s1 = quad_sum(hp[1][3]);
      if (q4 == 0) {
        const float b = p.use_viewdirs ? s_heads[640] : s_heads[1027];
        if (lrb + r0 < nrows) grid.sigma[row_begin + lrb + r0] = s0 + b;
        if (lrb + r1 < nrows) grid.sigma[row_begin + lrb + r1] = s1 + b;
      }
      continue;
    }
    // ---- heads: full row sums over the quad -> raw rows of the tile -> compositing ----
    ph.start();
    float raw[2][4];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int k = 0; k < 4; ++k) raw[h][k] = quad_sum(hp[h][k]);
    const uint32_t a_raw = sb + FWD_RAW + (uint32_t)(64 * w) * 16u;
    if (q4 == 0) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float4 o;
        if (p.use_viewdirs) o = make_float4(raw[h][0] + s_heads[641], raw[h][1] + s_heads[642], raw[h][2] + s_heads[643], raw[h][3] + s_heads[640]);
        else o = make_float4(raw[h][0] + s_heads[1024], raw[h][1] + s_heads[1025], raw[h][2] + s_heads[1026], raw[h][3] + s_heads[1027]);
        sts128(a_raw + (uint32_t)(h ? r1 : r0) * 16u, o);
      }
    }
    wg_sync();
    if (wq < 2) {
      const int tr = 32 * wq + lane;                              // row of the warpgroup
      const int lr = lrb + tr;
      const bool valid = lr < nrows;
      const int rl = (valid ? lr : nrows - 1) / p.S;
      long long n_ray = ray0 + rl;
      if (n_ray > p.N - 1) n_ray = p.N - 1;
      if (n_ray < 0) n_ray = 0;
      composite_rows(p, lds128(a_raw + (uint32_t)tr * 16u), valid, lr, rl, n_ray, row_begin, st, X, 2 * w + wq, lane, a_carry);
    }
    ph.stop(PH_COMPOSITOR);
  }
  if (EMIT && t == 0) ptx::bulk_wait_all();
  ph.flush(w, t);
}

template <bool EMIT>
__global__ void __launch_bounds__(TC_THREADS, 1) march_wg_kernel(const MarchParams p, const TrainSaveDev sv) {
  march_pass<EMIT, false>(p, sv, nullptr);
}

// precision TC_SPLIT: fp32-class results from three fp16 MMAs per K-step (inference only; wscale: the split image's scales)
__global__ void __launch_bounds__(TC_THREADS, 1) march_split_kernel(const MarchParams p, const float* __restrict__ wscale) {
  march_pass<false, true>(p, TrainSaveDev{}, wscale);
}

// precision TC_SPLIT in training mode: march_split_kernel's outputs, bit for bit, plus the split records (hi record, then lo
// record, per tile; mask bits = signs of the split fp32 pre-activations) that the split backward reads
__global__ void __launch_bounds__(TC_THREADS, 1) march_split_train_kernel(const MarchParams p, const TrainSaveDev sv, const float* __restrict__ wscale) {
  march_pass<true, true>(p, sv, wscale);
}

// The density grid (nerf_b200_density_grid): sigma on the points of `g`, precision TC_FP16 on the fp16 image, TC_SPLIT (wscale
// the split image's scales) on the split image.  The forward's shared-memory map; the raw rows, carry and the ring stages of
// the view layers go unused.
static_assert(FWD_ALLOC <= 227 * 1024, "the density pass's shared-memory map exceeds the per-block limit");
__global__ void __launch_bounds__(TC_THREADS, 1) density_wg_kernel(const MarchParams p, const DensityGrid g) {
  march_pass<false, false, true>(p, TrainSaveDev{}, nullptr, g);
}
__global__ void __launch_bounds__(TC_THREADS, 1) density_split_kernel(const MarchParams p, const DensityGrid g, const float* __restrict__ wscale) {
  march_pass<false, true, true>(p, TrainSaveDev{}, wscale, g);
}

}  // namespace nb
