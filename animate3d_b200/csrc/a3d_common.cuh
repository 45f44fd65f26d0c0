// animate3d_b200 -- sm_90a device helpers: mbarrier, TMA (cp.async.bulk.tensor), wgmma fences and descriptors.
// Everything here is inline PTX for sm_90a; there is no other backend.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdint.h>

namespace a3d {

// ---------------------------------------------------------------------------------------------------------------
// small utilities
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Spin on the barrier phase.  A pipeline bug would otherwise hang the GPU forever; after ~4 s of waiting the kernel
// traps so that the host sees a launch failure instead (the check costs nothing on the fast path).  No printf here: a call
// inside the wgmma main loops would make ptxas serialise the asynchronous MMAs.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 8000000000ll) __trap();
  }
}

// ---------------------------------------------------------------------------------------------------------------
// TMA: every tensor map in this library is rank-5 (unused trailing dims have extent 1)
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
        "r"(c3), "r"(c4)
      : "memory");
}
// generic-proxy writes to smem (st.shared) -> visible to the async proxy (wgmma / TMA reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// 32-byte global accesses as two 16-byte vector instructions (sm_90 has no 256-bit LDG / STG): the pair still covers one
// whole 32-byte sector per lane
__device__ __forceinline__ void st_global_256(void* ptr, const uint32_t* r) {
  asm volatile("st.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(ptr), "r"(r[0]), "r"(r[1]), "r"(r[2]), "r"(r[3]) : "memory");
  asm volatile("st.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(reinterpret_cast<uint8_t*>(ptr) + 16), "r"(r[4]), "r"(r[5]),
               "r"(r[6]), "r"(r[7])
               : "memory");
}

// single-instruction math used by the softmax code
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  uint32_t d;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}
// ---------------------------------------------------------------------------------------------------------------
// wgmma (sm_90a warpgroup MMA): fences, commit / wait, shared-memory matrix descriptors
// ---------------------------------------------------------------------------------------------------------------
// Accumulator registers touched by ordinary code must be fenced before the next wgmma reads them.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an asynchronous wgmma (register operands only)
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Shared-memory matrix descriptor, SWIZZLE_128B (bit layout: PTX ISA, "Matrix Descriptor Format" of wgmma).  Addresses and
// offsets are encoded >> 4; tiles are 1024-byte aligned, so the base-offset field stays 0.
//   K-major operand  : tile = R rows x 64 halves (128 B/row), 8-row groups 1024 B apart  -> SBO = 1024, LBO unused (1)
//   MN-major operand : atom = 64 (MN, contiguous) x 8 (K) halves = 1024 B; next 8 K-rows at SBO = 1024;
//                      next 64 MN elements at LBO = bytes of one TMA box (rows * 128 B)
// Stepping 16 halves along K inside a K-major atom adds 32 B to the start address (+2 in the encoded field).
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;  // layout_type = SWIZZLE_128B
  return d;
}

// warp-level MMA (fp16 x fp16 -> fp32), used where a problem is far below a 64-row warpgroup tile (16-frame temporal
// attention, 77-key text cross-attention)
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

}  // namespace a3d
