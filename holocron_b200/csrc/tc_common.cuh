// sm_90a building blocks for the tensor-core kernels: mbarrier, TMA (tiled + im2col), wgmma fences and
// shared-memory matrix descriptors. Inline PTX only.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "wgmma.cuh"

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t.reg .b32 R;\n\t"
      "elect.sync R|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier -------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
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
      "selp.b32 %0, 1, 0, P;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a protocol bug becomes a trap (visible launch failure) instead of a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) { asm volatile("trap;"); }
  }
}

// ---- TMA ------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// im2col-mode load of a 4-D NHWC tensor (dims C, W, H, N): `pixelsPerColumn` output pixels starting at
// base pixel (w, h, n) x `channelsPerPixel` channels starting at c, filter offset (off_w, off_h).
__device__ __forceinline__ void tma_load_im2col_4d(const CUtensorMap* m, uint64_t* bar, void* dst, int c, int w, int h,
                                                   int n, uint16_t off_w, uint16_t off_h) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n),
      "h"(off_w), "h"(off_h)
      : "memory");
}

// ---- wgmma -----------------------------------------------------------------------------------
// Ordering of the accumulator registers against the asynchronous warpgroup MMAs (all four are warpgroup-wide).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across a wgmma wait
template <int N>
__device__ __forceinline__ void fence_regs(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}

// ---- register reallocation between warpgroups ------------------------------------------------
// Warpgroup-wide (every thread of the warpgroup executes it). A warpgroup that only issues TMA hands registers back to the
// SM's pool so that the MMA warpgroups of the same CTA can hold wider accumulators. N: a multiple of 8 in [24, 256];
// the sum over the CTA's warpgroups of 128 * N must fit in the 64 K registers of an SM.
template <int N>
__device__ __forceinline__ void regs_release() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void regs_acquire() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// ---- descriptors ----------------------------------------------------------------------------
// Shared-memory matrix descriptor of wgmma (sm_90):
//   [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [49,52) base offset | [62,64) layout (1 = 128B swizzle)
// The 128-byte swizzle is a function of the absolute shared-memory address (the TMA writes it that way), so a
// descriptor may start at any 128-byte row of a 1024-byte aligned buffer and advancing along K inside a row is a plain
// address add: the low word carries the address, the high word (SBO, layout) stays fixed.
//   K-major operand (rows = M or N, 128-byte rows of 64 K elements): SBO = 1024 (8-row atom), LBO unused.
//   MN-major operand (rows = K, 128-byte rows of 64 M/N elements): SBO = 1024 (next 8 K rows), LBO = distance
//   between 64-element atoms along M/N.
__device__ __forceinline__ uint32_t desc_hi(uint32_t sbo_bytes) { return ((sbo_bytes >> 4) & 0x3FFF) | (1u << 30); }
__device__ __forceinline__ uint32_t desc_lo(uint32_t saddr, uint32_t lbo_bytes) {
  return ((saddr >> 4) & 0x3FFF) | (((lbo_bytes >> 4) & 0x3FFF) << 16);
}
__device__ __forceinline__ uint64_t make_desc(uint32_t lo, uint32_t hi) { return ((uint64_t)hi << 32) | lo; }

// Accumulator fragment of an m64nN wgmma: register i of thread t holds row  16*(warp of t) + lane/4 (+8 when i & 2)
// and column  8*(i/4) + 2*(lane%4) + (i & 1)  of the warpgroup's 64-row tile.
__device__ __forceinline__ int frag_row(int t) { return ((t >> 5) & 3) * 16 + ((t & 31) >> 2); }
__device__ __forceinline__ int frag_col(int t) { return (t & 3) * 2; }

// ---- MMA issue ------------------------------------------------------------------------------
// One commit group: KS k-steps of width N issued straight-line between a fence and a commit. Every fence -> commit
// region of a kernel must be such a sequence; a predicate, a loop with a run-time trip count or a branch between
// different MMAs inside the region makes ptxas serialise all wgmmas of the kernel (notes C7519 / C7520).
// Descriptor low words advance by `step` per k-step; the first k-step uses `scale_first` (0 = overwrite).
template <int N, int KS, int TA, int TB>
__device__ __forceinline__ void wgmma_group(float* d, uint32_t a_lo, uint32_t b_lo, uint32_t step, uint32_t dhi,
                                            uint32_t scale_first) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < KS; ++k)
    wgmma<N, TA, TB>(d, make_desc(a_lo + k * step, dhi), make_desc(b_lo + k * step, dhi), k ? 1u : scale_first);
  wgmma_commit();
}
// The same for a 64-channel block with a run-time k-step count ks in 1..4 (a partial last channel block): the switch
// picks a whole region, so each region stays straight-line.
template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_group_ks(int ks, float* d, uint32_t a_lo, uint32_t b_lo, uint32_t step,
                                               uint32_t dhi, uint32_t scale_first) {
  switch (ks) {
    case 1: wgmma_group<N, 1, TA, TB>(d, a_lo, b_lo, step, dhi, scale_first); break;
    case 2: wgmma_group<N, 2, TA, TB>(d, a_lo, b_lo, step, dhi, scale_first); break;
    case 3: wgmma_group<N, 3, TA, TB>(d, a_lo, b_lo, step, dhi, scale_first); break;
    default: wgmma_group<N, 4, TA, TB>(d, a_lo, b_lo, step, dhi, scale_first); break;
  }
}

}  // namespace tc
