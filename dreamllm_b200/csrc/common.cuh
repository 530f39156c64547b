// Shared sm_90a device helpers: mbarrier, TMA, wgmma wrappers (raw PTX).
// Everything here is hand-written for this repo; encodings follow the PTX ISA / the public
// CUTLASS headers' documentation of the GMMA descriptors.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace dllm {

typedef __nv_bfloat16 bf16;

#ifndef DLLM_WATCHDOG
#define DLLM_WATCHDOG 1  // bounded mbarrier waits: a protocol bug traps instead of hanging the GPU
#endif

// ----------------------------------------------------------------------------- misc
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .b32 rx;\n\t.reg .pred px;\n\t"
      "elect.sync rx|px, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, px;\n\t}"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ----------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
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
// Bounded wait (DLLM_WATCHDOG=1, the default): a protocol bug traps after ~2 s instead of hanging the GPU.  The slow path holds no
// function call (no printf): ptxas serialises every wgmma of a kernel whose wgmma pipeline crosses a call (C7510), and the consumers
// wait on the operand ring while their previous K block's wgmma group is still in flight.  `tag` names the wait site in the SASS
// (the immediate of the trap's preceding move) for reading a core dump; it costs nothing at run time.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag = 0) {
#if DLLM_WATCHDOG
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0xfff) == 0 && clock64() - t0 > 4000000000LL) {  // ~2 s
      asm volatile("{\n\t.reg .b32 t;\n\tmov.b32 t, %0;\n\ttrap;\n\t}" ::"r"(tag));
    }
  }
#else
  (void)tag;
  while (!mbar_try_wait(bar, parity)) {
  }
#endif
}

// ----------------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2D tile load global -> this CTA's smem, completion on this CTA's mbarrier
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
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
// four 8 x 8 b16 blocks from the mma accumulator fragment layout (thread i: row i / 4, elements 2 (i % 4), + 1 of each block) to shared
// memory; lanes 8 b .. 8 b + 7 give the addresses of the rows of block b (16 bytes each).  No "memory" clobber: volatile keeps it in
// order with the fences and barriers around it, and global loads may move across it.  Nothing reads what it wrote through C++.
__device__ __forceinline__ void stmatrix_x4(uint32_t saddr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(r0), "r"(r1), "r"(r2), "r"(r3));
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ----------------------------------------------------------------------------- wgmma (sm_90a warpgroup MMA)
// Shared-memory matrix descriptor of the sm_90 GMMA, 128-byte swizzle (layout type 1):
//   bits [0,14)  start address >> 4       bits [16,30) leading byte offset >> 4
//   bits [32,46) stride byte offset >> 4  bits [62,64) layout type
// K-major operand (rows x 64 bf16 per 128-byte line, 8-row swizzle atoms of 1024 B):
//   SBO = 1024 (distance between 8-row groups); LBO unused (16).  Advance 32 B per K = 16 step.
// MN-major operand (64 mn-elements per 128-byte line, one line per k; boxes of [64 mn x BK k]):
//   LBO = distance between 64-element mn groups (box bytes); SBO = 1024 (8 k-lines).  Advance 2048 B per K = 16 step.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// descriptor of K step `ks` (16 elements) of a 128B-swizzled tile
//   K-major : tile = [K/64 chunks][rows][128 B]; chunk_stride = bytes between 64-wide K chunks
//   MN-major: tile = [MN/64 groups][K lines][128 B]; chunk_stride = bytes between 64-wide MN groups (LBO)
__device__ __forceinline__ uint64_t op_desc(uint32_t base, bool mn, uint32_t chunk_stride, int ks) {
  return mn ? make_smem_desc(base + ks * 2048u, chunk_stride, 1024u)
            : make_smem_desc(base + (ks >> 2) * chunk_stride + (ks & 3) * 32u, 16u, 1024u);
}
// wgmma_fence orders this warpgroup's register writes of accumulators / A fragments before the next wgmma reads them
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// per-warpgroup register budget (the TMA warpgroup hands registers to the MMA warpgroups)
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}

// The 8-element vector copies of the HBM-bound kernels are 128-bit accesses, which fault on addresses that are not 16-byte aligned:
// the host wrappers reject such pointers up front (DLLM_ERR_ALIGN).
#define DLLM_REQUIRE_ALIGN16(...)                                                        \
  do {                                                                                   \
    const void* dllm_ps_[] = {__VA_ARGS__};                                              \
    for (const void* dllm_p_ : dllm_ps_)                                                 \
      if (reinterpret_cast<uintptr_t>(dllm_p_) & 15u) return -2; /* DLLM_ERR_ALIGN */    \
  } while (0)

// ----------------------------------------------------------------------------- small math helpers
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace dllm

// ----------------------------------------------------------------------------- 3D TMA (batched [B, S, cols] views)
namespace dllm {
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
// 4D tile loads ([N, H, W, C] activations for the implicit-GEMM 3x3 convolution; OOB coordinates zero-fill = padding)
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
}  // namespace dllm
