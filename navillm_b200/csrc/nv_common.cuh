// navillm_b200 — shared device-side primitives for the sm_90a kernels.
//
// Thin inline-PTX wrappers for the Hopper async machinery used by every hot
// kernel in this package: mbarrier, TMA (cp.async.bulk.tensor), warpgroup MMA
// (wgmma ordering and shared-memory descriptors; the MMA wrappers themselves are
// in nv_wgmma.cuh).  Nothing here is a port of reference code: the reference
// (zd11024/NaviLLM) ships no native sources (SURVEY.md §2a).
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "nv_wgmma.cuh"

namespace nv {

// ----------------------------------------------------------------------------------------------
// small helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() {
  uint32_t l;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
  return l;
}
__host__ __device__ constexpr uint32_t ceil_div_u32(uint32_t a, uint32_t b) { return (a + b - 1) / b; }

// round-to-nearest-even fp32 -> bf16 bits, packed pair (lo = a, hi = b)
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// Programmatic dependent launch (PDL).  A kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may
// start while its predecessor in the stream is still running: `griddep_wait` blocks until the predecessor grid has
// completed and its memory is visible (every thread calls it before its first read of predecessor-produced data and
// before its first global write); `griddep_launch` lets the NEXT kernel's CTAs be scheduled early.  Both are no-ops when
// the kernel was launched without the attribute.
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// explicit shared-window accesses (32-bit addresses: STS/LDS instead of generic ST.E/LD.E through 64-bit pointers)
__device__ __forceinline__ void sts128(uint32_t saddr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ uint2 lds64(uint32_t saddr) {
  uint2 v;
  asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(saddr) : "memory");
  return v;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps after ~2 s (error surfaces on the host as a launch failure)
// instead of hanging the GPU box.
#ifndef NV_MBAR_TIMEOUT_CYCLES
#define NV_MBAR_TIMEOUT_CYCLES (4000000000ll)
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 255u) == 0 && clock64() - t0 > NV_MBAR_TIMEOUT_CYCLES) {
      printf("navillm_b200: mbarrier timeout block (%d,%d) thread %d bar@%u parity %u\n", (int)blockIdx.x,
             (int)blockIdx.y, (int)threadIdx.x, smem_u32(bar), parity);
      __trap();
    }
  }
}

// generic-proxy smem writes -> visible to the async proxy (TMA stores / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ----------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0,
                                            int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0,
                                            int32_t c1, int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------------------------
// warpgroup MMA (wgmma): ordering and shared-memory matrix descriptors
// ----------------------------------------------------------------------------------------------
// wgmma_fence before the first wgmma that reads accumulator / A registers written by ordinary instructions;
// wgmma_commit closes the group of wgmmas issued so far; wgmma_wait<N> returns when at most N groups are pending
// (their accumulators are then readable and their shared-memory operands may be overwritten).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// The accumulator registers are not visible to the compiler as wgmma operands between issue and wait: this pins them.
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// One lane of a converged warp (TMA issue from code the whole warp runs keeps the operands in uniform registers).
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred e;\n\telect.sync _|e, 0xffffffff;\n\tselp.u32 %0, 1, 0, e;\n\t}" : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ uint32_t warp_id_uniform() { return __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0); }

// Named barrier over `count` threads (multiple of 32); id 0 is __syncthreads.
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ----------------------------------------------------------------------------------------------
// thread-block clusters: barrier over every thread of every CTA, and a read-modify-write of a float in the
// shared memory of another CTA (distributed shared memory)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// *(float at shared address `saddr` in CTA `cta` of the cluster) += v   (the caller guarantees a single writer)
__device__ __forceinline__ void dsmem_add_f32(uint32_t saddr, uint32_t cta, float v) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t.reg .f32 x;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "ld.shared::cluster.f32 x, [ra];\n\t"
      "add.f32 x, x, %2;\n\t"
      "st.shared::cluster.f32 [ra], x;\n\t}"
      ::"r"(saddr), "r"(cta), "f"(v)
      : "memory");
}

// sm_90 shared-memory matrix descriptor, 128-byte swizzle (PTX ISA "Matrix Descriptor Format" of wgmma):
//   bits [0,14) start address >> 4   [16,30) leading byte offset >> 4   [32,46) stride byte offset >> 4
//   [62,64) layout type (1 = SWIZZLE_128B)
// K-major tile (rows of 64 bf16 / 32 fp32 = 128 B, 8-row swizzle atoms): SBO = 1024, LBO unused; a 32-byte K step is +2.
// MN-major tile (rows = K index, 64 MN elements = 128 B per row, one 64-wide MN atom after the other): SBO = 1024
// (next 8 K rows), LBO = bytes between consecutive 64-wide MN atoms; a 16-row K step is +128.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFFu);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// Byte offset of 16-byte chunk `chunk` (0..7) in row `row` of a 128-byte-swizzled tile whose rows are
// 128 B and whose base is 1024-byte aligned (the layout TMA SWIZZLE_128B writes and wgmma reads).
__device__ __forceinline__ uint32_t sw128_offset(uint32_t row, uint32_t chunk) {
  return row * 128u + ((chunk ^ (row & 7u)) << 4);
}

}  // namespace nv
