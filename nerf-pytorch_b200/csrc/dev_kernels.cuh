// dev_kernels.cuh -- bring-up and measurement kernels, NOT part of the product library: wgmma self-test GEMMs (K-major
// and MN-major operand encodings of the fused pass and of the weight gradient) and the HBM stream probes.  Compiled only
// into libnerf_b200_dev.so (capi_dev.cu).
#pragma once
#include "fused_tc.cuh"
#include "fused_wg.cuh"

namespace nb {

// ---------------------------------------------------------------------------------------------
// self-test GEMM: out[128,N] = A[128,K] * W[N,K]^T through exactly the operand layouts and descriptors the fused pass uses
// (A: 64-row K-blocks of 8 KB, SWIZZLE_128B, written by threads; W: packed [N x 32] SWIZZLE_64B chunks by bulk copy; fp16
// operands, fp32 accumulation).  1 CTA = 2 warpgroups, each on 64 rows.
// ---------------------------------------------------------------------------------------------
template <int N>
__device__ __forceinline__ void selftest_gemm_body(const float* A, const uint8_t* chunks, int K, float* out, uint32_t sb) {
  constexpr uint32_t WST = 65536, BAR = WST + 131072;
  const int w = threadIdx.x >> 7, t = threadIdx.x & 127, wq = t >> 5, lane = t & 31;
  const uint32_t act = sb + (uint32_t)w * 32768u;
  // rows 64 w .. of A as fp16 into the warpgroup's K-blocks
  for (int i = t; i < 64 * (K / 2); i += 128) {
    const int r = i / (K / 2), c = 2 * (i % (K / 2));
    const float* a = A + (size_t)(64 * w + r) * K + c;
    ptx::st_shared_b32(act + half_off(r, c), ptx::cvt_f16x2(a[0], a[1]));
  }
  const uint32_t cb = (uint32_t)N * 64u * (uint32_t)(K / 32);
  if (threadIdx.x == 0) {
    ptx::mbar_init(sb + BAR, 1);
    ptx::fence_mbar_init();
  }
  ptx::fence_proxy_async_smem();
  __syncthreads();
  if (threadIdx.x == 0) {
    ptx::mbar_arrive_expect_tx(sb + BAR, cb);
    ptx::bulk_g2s(sb + WST, chunks, cb, sb + BAR);
  }
  ptx::mbar_wait(sb + BAR, 0);
  float acc[N / 2];
  ptx::wgmma_fence();
  for (int c = 0; c < K / 32; ++c) {
    const uint64_t ad = desc_act(act + (uint32_t)(c >> 1) * 8192u + (uint32_t)(c & 1) * 64u);
    const uint64_t bd = desc_w(sb + WST + (uint32_t)c * N * 64u);
    mma_chunk(acc, ad, bd, c > 0 ? 1u : 0u);
  }
  ptx::wgmma_commit();
  ptx::wgmma_wait<0>();
  ptx::fence_regs(acc);
  const int r0 = 64 * w + 16 * wq + (lane >> 2), q4 = lane & 3;
  for (int j = 0; j < N / 8; ++j) {
    const int c = 8 * j + 2 * q4;
    out[(size_t)r0 * N + c] = acc[4 * j]; out[(size_t)r0 * N + c + 1] = acc[4 * j + 1];
    out[(size_t)(r0 + 8) * N + c] = acc[4 * j + 2]; out[(size_t)(r0 + 8) * N + c + 1] = acc[4 * j + 3];
  }
}
__global__ void __launch_bounds__(256, 1) selftest_gemm_kernel(const float* __restrict__ A, const uint8_t* __restrict__ chunks,
                                                               int K, int N, float* __restrict__ out) {
  const uint32_t sb = ptx::smem_u32(tc_smem);
  if ((sb & 1023u) != 0) __trap();
  if (N == 256) selftest_gemm_body<256>(A, chunks, K, out, sb);
  else selftest_gemm_body<128>(A, chunks, K, out, sb);
}

// ---------------------------------------------------------------------------------------------
// "TN" self-test for the weight-gradient GEMM of the backward: out[256,256] = X^T Y with X, Y [128 rows, 256] given as
// activation tiles (row = sample, K-blocks of 64 columns x 128 rows, SWIZZLE_128B) and read by the MMA as MN-MAJOR operands:
// A = X viewed [M = column, K = row], B = Y viewed [N = column, K = row].  The canonical MN-major SWIZZLE_128B atom is 64
// contiguous MN elements x 8 K rows = the same physical 1 KB atom as the K-major one, so no re-layout is needed:
// LBO = stride between 64-column groups (16 KB: the K-block stride), SBO = stride between 8-row groups (1 KB).  lbo / sbo
// are arguments so that one GPU run can confirm the encoding.  1 CTA = 1 warpgroup, one 64-row block of out at a time.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128, 1) selftest_gemm_tn_kernel(const float* __restrict__ X, const float* __restrict__ Y,
                                                                  float* __restrict__ out, uint32_t lbo, uint32_t sbo) {
  const uint32_t sb = ptx::smem_u32(tc_smem);
  if ((sb & 1023u) != 0) __trap();
  constexpr uint32_t XT = 0, YT = 65536;
  const int t = threadIdx.x, wq = t >> 5, lane = t & 31;
  for (int i = t; i < 128 * 128; i += 128) {
    const int r = i >> 7, c = 2 * (i & 127);
    const uint32_t o = (uint32_t)(c >> 6) * 16384u + (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((((c & 63) >> 3) ^ (r & 7)) << 4) + (c & 7) * 2);
    ptx::st_shared_b32(sb + XT + o, ptx::cvt_f16x2(X[r * 256 + c], X[r * 256 + c + 1]));
    ptx::st_shared_b32(sb + YT + o, ptx::cvt_f16x2(Y[r * 256 + c], Y[r * 256 + c + 1]));
  }
  ptx::fence_proxy_async_smem();
  __syncthreads();
  float acc[128];
  for (int mb = 0; mb < 4; ++mb) {
    ptx::wgmma_fence();
    for (int k = 0; k < 8; ++k) {
      const uint64_t ad = ptx::gmma_desc(sb + XT + mb * 16384 + k * 2048, lbo, sbo, ptx::GMMA_SW128);
      const uint64_t bd = ptx::gmma_desc(sb + YT + k * 2048, lbo, sbo, ptx::GMMA_SW128);
      ptx::wgmma_m64n256k16<1, 1>(acc, ad, bd, k > 0 ? 1u : 0u);
    }
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_regs(acc);
    const int r0 = 64 * mb + 16 * wq + (lane >> 2), q4 = lane & 3;
    for (int j = 0; j < 32; ++j) {
      const int c = 8 * j + 2 * q4;
      out[r0 * 256 + c] = acc[4 * j]; out[r0 * 256 + c + 1] = acc[4 * j + 1];
      out[(r0 + 8) * 256 + c] = acc[4 * j + 2]; out[(r0 + 8) * 256 + c + 1] = acc[4 * j + 3];
    }
  }
}

// ---- HBM stream probes: what a pure read / pure write / mixed stream reaches on this GPU (context for the training kernels,
// which are bound by record writes (forward, dgrad) or record reads (wgrad)) -----------------------------------------------
// mode 0: read n 16-byte words (xor-reduced, result kept alive); 1: write; 2: read `src`, write `dst` (copy)
__global__ void __launch_bounds__(512) hbm_stream_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, size_t n, int mode, uint4* sink) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint4 acc = make_uint4(0u, 0u, 0u, 0u);
  if (mode == 0) {
    for (; i + 7 * stride < n; i += 8 * stride) {
      uint4 v[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = __ldcs(src + i + k * stride);
#pragma unroll
      for (int k = 0; k < 8; ++k) { acc.x ^= v[k].x; acc.y ^= v[k].y; acc.z ^= v[k].z; acc.w ^= v[k].w; }
    }
    for (; i < n; i += stride) { const uint4 v = __ldcs(src + i); acc.x ^= v.x; acc.y ^= v.y; acc.z ^= v.z; acc.w ^= v.w; }
    if ((acc.x ^ acc.y ^ acc.z ^ acc.w) == 0x9e3779b9u) *sink = acc;
  } else if (mode == 1) {
    const uint4 v = make_uint4((uint32_t)i, 1u, 2u, 3u);
    for (; i < n; i += stride) __stcs(dst + i, v);
  } else {
    for (; i + 3 * stride < n; i += 4 * stride) {
      uint4 v[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] = __ldcs(src + i + k * stride);
#pragma unroll
      for (int k = 0; k < 4; ++k) __stcs(dst + i + k * stride, v[k]);
    }
    for (; i < n; i += stride) __stcs(dst + i, __ldcs(src + i));
  }
}


// ---- per-SM DRAM streaming probe: what ONE CTA per SM moves between HBM and shared memory / registers with each mechanism ----
// Every CTA streams its own disjoint `bytes_per_cta` region (no L2 reuse when the buffer is much larger than L2).
//   mode 0: cp.async.bulk global->shared through a ring of `stages` x `chunk` bytes (one producer lane, one consumer warp)
//   mode 1: cp.async 16-byte copies (LDGSTS) by 128 producer threads into the same ring, completion through
//           cp.async.mbarrier.arrive.noinc
//   mode 2: cp.async.bulk shared->global of `chunk` bytes, at most `stages` bulk groups pending (wait_group.read)
//   mode 3: st.global.v4 by 512 threads          mode 4: ld.global.v4 by 512 threads (8 loads in flight per thread)
// shared_bytes != 0 (mode 0 only): every CTA streams the SAME first `shared_bytes` of `buf`, cyclically, for bytes_per_cta in
// all -- an L2-resident stream, as the weight chunks of the fused forward (every CTA walks one 1 179 648-byte chunk sequence).
// out[blockIdx.x] = clock cycles of the CTA's stream.
constexpr int DSP_THREADS = 512;
__global__ void __launch_bounds__(DSP_THREADS, 1) dram_stream_probe_kernel(uint8_t* __restrict__ buf, unsigned long long bytes_per_cta, int chunk, int stages,
                                                                           int mode, long long* out, int scatter, unsigned long long shared_bytes) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const uint32_t sb = ptx::smem_u32(smem);
  const uint32_t BAR = (uint32_t)stages * (uint32_t)chunk;
  const int warp = threadIdx.x >> 5;
  uint8_t* base = shared_bytes ? buf : buf + (size_t)blockIdx.x * bytes_per_cta;
  const int n = (int)(bytes_per_cta / (unsigned)chunk);
  // scatter: chunk i of the CTA's region is visited in a strided order (i * 37 mod n: successive chunks ~600 KB apart for 16 KB
  // chunks), like the per-tile records of the training kernels, instead of front to back
  auto at = [&](int i) -> size_t {
    if (shared_bytes) return ((size_t)i * (size_t)chunk) % (size_t)shared_bytes;
    return (size_t)(scatter ? (int)(((long long)i * 37) % n) : i) * (size_t)chunk;
  };
  if (threadIdx.x == 0) {
    for (int i = 0; i < stages; ++i) { ptx::mbar_init(sb + BAR + 8 * i, mode == 1 ? 128 : 1); ptx::mbar_init(sb + BAR + 128 + 8 * i, 1); }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  const long long t0 = clock64();
  if (mode == 0 || mode == 1) {
    if (mode == 0 && warp == 0) {
      uint32_t stage = 0, ph = 0;
      for (int i = 0; i < n; ++i) {
        ptx::mbar_wait(sb + BAR + 128 + 8 * stage, ph ^ 1);
        if (ptx::elect_one()) {
          ptx::mbar_arrive_expect_tx(sb + BAR + 8 * stage, chunk);
          for (int o = 0; o < chunk; o += 8192) ptx::bulk_g2s(sb + stage * chunk + o, base + at(i) + o, (chunk - o) < 8192 ? (chunk - o) : 8192, sb + BAR + 8 * stage);
        }
        __syncwarp();
        if (++stage == (uint32_t)stages) { stage = 0; ph ^= 1; }
      }
    } else if (mode == 1 && warp < 4) {
      uint32_t stage = 0, ph = 0;
      for (int i = 0; i < n; ++i) {
        ptx::mbar_wait(sb + BAR + 128 + 8 * stage, ph ^ 1);
        const uint8_t* src = base + (size_t)i * chunk;
        for (int o = threadIdx.x * 16; o < chunk; o += 128 * 16)
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(sb + stage * chunk + o), "l"(src + o) : "memory");
        asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" :: "r"(sb + BAR + 8 * stage) : "memory");
        if (++stage == (uint32_t)stages) { stage = 0; ph ^= 1; }
      }
    } else if (warp == 4) {
      uint32_t stage = 0, ph = 0;
      for (int i = 0; i < n; ++i) {
        ptx::mbar_wait(sb + BAR + 8 * stage, ph);
        if (ptx::elect_one()) ptx::mbar_arrive(sb + BAR + 128 + 8 * stage);
        __syncwarp();
        if (++stage == (uint32_t)stages) { stage = 0; ph ^= 1; }
      }
    }
  } else if (mode == 2) {
    if (threadIdx.x == 0) {
      ptx::fence_proxy_async_smem();
      for (int i = 0; i < n; ++i) {
        for (int o = 0; o < chunk; o += 16384) ptx::bulk_s2g(base + at(i) + o, sb + (uint32_t)(i % stages) * chunk + o, (chunk - o) < 16384 ? (chunk - o) : 16384);
        ptx::bulk_commit();
        switch (stages) {
          case 1: asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); break;
          case 2: asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); break;
          case 3: asm volatile("cp.async.bulk.wait_group.read 2;" ::: "memory"); break;
          case 4: asm volatile("cp.async.bulk.wait_group.read 3;" ::: "memory"); break;
          default: asm volatile("cp.async.bulk.wait_group.read 7;" ::: "memory"); break;
        }
      }
      ptx::bulk_wait_all();
    }
  } else if (mode == 3) {
    uint4* d = reinterpret_cast<uint4*>(base);
    const size_t nw = bytes_per_cta / 16;
    const uint4 v = make_uint4(threadIdx.x, 1u, 2u, 3u);
    for (size_t i = threadIdx.x; i < nw; i += DSP_THREADS) __stcs(d + i, v);
  } else {
    const uint4* d = reinterpret_cast<const uint4*>(base);
    const size_t nw = bytes_per_cta / 16;
    uint4 acc = make_uint4(0u, 0u, 0u, 0u);
    size_t i = threadIdx.x;
    for (; i + 7 * DSP_THREADS < nw; i += 8 * DSP_THREADS) {
      uint4 v[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = __ldcs(d + i + k * DSP_THREADS);
#pragma unroll
      for (int k = 0; k < 8; ++k) { acc.x ^= v[k].x; acc.y ^= v[k].y; acc.z ^= v[k].z; acc.w ^= v[k].w; }
    }
    if ((acc.x ^ acc.y ^ acc.z ^ acc.w) == 0x9e3779b9u) out[gridDim.x] = acc.x;
  }
  __syncthreads();
  if (threadIdx.x == 0) out[blockIdx.x] = clock64() - t0;
}

}  // namespace nb
