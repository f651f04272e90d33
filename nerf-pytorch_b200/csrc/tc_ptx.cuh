// tc_ptx.cuh -- thin inline-PTX wrappers for sm_90a: mbarrier, bulk async copy (TMA engine, SASS UBLKCP), the warpgroup
// MMA (wgmma: fences, commit / wait groups, shared-memory matrix descriptors) and register-count hand-off (setmaxnreg).
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>
#include "wgmma_ops.cuh"

namespace nb {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier --------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) { }
}

// ---- proxy fences ----------------------------------------------------------------------------
// generic-proxy st.shared  ->  async-proxy (wgmma / bulk copy) readers
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- bulk async copy global -> shared (TMA engine, completes on an mbarrier) -------------------
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src_gmem, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst_smem), "l"(src_gmem), "r"(bytes), "r"(bar) : "memory");
}

// ---- bulk async copy shared -> global (TMA engine, bulk-group completion; per-thread groups) ------
__device__ __forceinline__ void bulk_s2g(void* dst_gmem, uint32_t src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(src_smem), "r"(bytes) : "memory");
}
// the same with an L2 eviction-priority hint (createpolicy): streaming records are written / read once
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void bulk_s2g_hint(void* dst_gmem, uint32_t src_smem, uint32_t bytes, uint64_t policy) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(dst_gmem), "r"(src_smem), "r"(bytes), "l"(policy) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all of this thread's committed groups have finished READING shared memory (the source may be overwritten)
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---- wgmma ordering ----------------------------------------------------------------------------
// before the first wgmma that reads accumulator registers written by ordinary instructions
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ---- shared-memory matrix descriptor (wgmma) ---------------------------------------------------
// K-major operands: SWIZZLE_128B rows of 128 B (64 fp16), 8-row atoms of 1024 B (SBO = 1024);
//                   SWIZZLE_64B  rows of  64 B (32 fp16), 8-row atoms of  512 B (SBO =  512);
// MN-major operands (SWIZZLE_128B): the same physical 1 KB atom read as 64 contiguous M (N) elements x 8 K rows;
//                   LBO = stride between 64-element groups along M (N), SBO = stride between 8-row groups along K.
constexpr uint64_t GMMA_SW128 = 1, GMMA_SW64 = 2, GMMA_SW32 = 3;
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint64_t layout_type) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);        // start address  [0,14)
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;    // LBO            [16,30)
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;    // SBO            [32,46)
  d |= layout_type << 62;                              // swizzle mode   [62,64)
  return d;
}

// ---- register hand-off between warpgroups (producer gives registers to the MMA warpgroups) ------
template <int R> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// one elected lane of a fully converged warp
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.b32 %0, 1, 0, P;\n\t}" : "=r"(pred));
  return pred != 0;
}

// ---- packing helpers ----------------------------------------------------------------------------
// {lo = a, hi = b} as fp16 pair with ReLU fused into the conversion
__device__ __forceinline__ uint32_t cvt_relu_f16x2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
__device__ __forceinline__ uint32_t cvt_f16x2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
// saturating variant (+-65504 instead of inf): loss-scaled gradients of the fp16 backward
__device__ __forceinline__ uint32_t cvt_sat_f16x2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t a) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(a) : "memory");
}
// four 8 x 8 fp16 matrices, register i of every lane into matrix i; lanes 8 i .. 8 i + 7 give the addresses of its 8 rows
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ uint32_t ld_shared_b32(uint32_t addr) {
  uint32_t v; asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory"); return v;
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

}  // namespace ptx
}  // namespace nb
