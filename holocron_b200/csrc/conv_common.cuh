// What the four tensor-core convolution units (conv_fprop.cu, conv_rows.cu, conv_wgrad.cu, conv_wgrad_rows.cu) share:
// the warp roles, the mbarrier ring position, the epilogue pieces that are the same in every kernel, the launch helper,
// the run-time tile-width dispatch and the internal entry points of the row-window kernels.
#pragma once
#include <cuda_runtime.h>
#include <type_traits>
#include "common.cuh"
#include "tc_common.cuh"
#include "tmap.cuh"

namespace conv {

// Warp roles: warpgroup 0 is the TMA producer, warpgroups 1-2 are the consumers (MMAs + epilogue).
constexpr int kThreads = 384;
constexpr int kConsumers = 256;

// Named barrier 1 over the two consumer warpgroups.
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// Position in a ring of n slots with one full and one empty mbarrier per slot: the consumers wait on full[stage] with
// `phase`, the producer waits on empty[stage] with `phase ^ 1` (the first pass finds every slot free). Pass k of the
// ring uses slot k % n with parity (k / n) & 1. The pipelined kernels step through it with next(); the row-window kernels,
// which take one slot per tile, position it from their tile counter with at() (one register live across the tile loop).
struct Ring {
  int stage = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ void next(int n) {
    if (++stage == n) { stage = 0; phase ^= 1; }
  }
  __device__ __forceinline__ static Ring at(int k, int n) { return Ring{k % n, (uint32_t)(k / n) & 1}; }
};

// ---- epilogue pieces --------------------------------------------------------------------------------------------------
// Residual add (+ ReLU) of one 16-byte chunk of 8 bf16 values, in fp32, rounded once.
__device__ __forceinline__ void add_residual16(uint4& val, const uint4& rv, bool relu) {
  __nv_bfloat162* a = reinterpret_cast<__nv_bfloat162*>(&val);
  const __nv_bfloat162* b = reinterpret_cast<const __nv_bfloat162*>(&rv);
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    float2 fa = __bfloat1622float2(a[jj]), fb = __bfloat1622float2(b[jj]);
    fa.x += fb.x; fa.y += fb.y;
    if (relu) { fa.x = hb::relu_nan(fa.x); fa.y = hb::relu_nan(fa.y); }
    a[jj] = __floats2bfloat162_rn(fa.x, fa.y);
  }
}

// Output-column statistics. Each thread keeps (sum0, sum1, sumsq0, sumsq1) of one column pair over a subset of the rows;
// accum_pair adds one staged bf16 pair to it.
__device__ __forceinline__ void accum_pair(float4& s, const uint8_t* staged) {
  const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(staged));
  s.x += f.x; s.y += f.y; s.z = fmaf(f.x, f.x, s.z); s.w = fmaf(f.y, f.y, s.w);
}
// (sum, sum of squares) of column c: the row subsets' partials, scratch[rg * npairs + c / 2] for rg < rgs, added in
// rg order (deterministic).
__device__ __forceinline__ float2 fold_stats(const float4* scratch, int rgs, int npairs, int c) {
  const int pr = c >> 1, hi = c & 1;
  float sv = 0.f, qv = 0.f;
  for (int rg = 0; rg < rgs; ++rg) {
    const float4 v = scratch[rg * npairs + pr];
    sv += hi ? v.y : v.x;
    qv += hi ? v.w : v.z;
  }
  return make_float2(sv, qv);
}
// The statistics buffer read by the training BatchNorm: float [slots][Cout][2] = (sum, sum of squares) partials. Every
// (slot, channel) entry is written exactly once, zeros included, so the reader adds all slots without a memset.
__device__ __forceinline__ void store_stats(float* stats, int slot, int Cout, int channel, float2 v) {
  *reinterpret_cast<float2*>(stats + ((size_t)slot * Cout + channel) * 2) = v;
}

// ---- host side ----------------------------------------------------------------------------------------------------------
// Launches kKernel with kThreads threads and smem_bytes of dynamic shared memory, and counts the launch. The kernel's
// dynamic shared-memory limit is raised to 227 KiB on its first launch.
template <auto kKernel, typename... Args>
cudaError_t launch(int grid, size_t smem_bytes, cudaStream_t stream, const Args&... args) {
  static const cudaError_t attr =
      cudaFuncSetAttribute(kKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  if (attr != cudaSuccess) return attr;
  kKernel<<<grid, kThreads, smem_bytes, stream>>>(args...);
  g_hb_launches.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError();
}

// Calls f(std::integral_constant<int, W>{}) for the run-time width w = W in {kStep, 2 kStep, ..., kMax}: one kernel
// instantiation per width. Any other w returns cudaErrorInvalidValue.
template <int kStep, int kMax, int W = kStep, typename F>
cudaError_t dispatch_width(int w, F&& f) {
  if (w == W) return f(std::integral_constant<int, W>{});
  if constexpr (W + kStep <= kMax) return dispatch_width<kStep, kMax, W + kStep>(w, f);
  else return cudaErrorInvalidValue;
}

}  // namespace conv

// Row-window kernels for stride-1 3x3 layers (conv_rows.cu, conv_wgrad_rows.cu), behind the public entry points. Both
// return 0 after a launch, cudaErrorNotSupported when the shape is not eligible (nothing launched: the caller uses the
// generic kernel), or the launch's own error.
//
// y = conv3x3(x, w) + sum_{e < nextra} conv1x1(xe[e], we[e]) (+ bias, residual, ReLU): up to two extra [N,H,W,Cin]
// sources with [Cout,1,1,Cin] filters in the same accumulator. stats: optional output-column statistics, with
// *stat_slots set to the slot count.
int hb_conv_rows_try(const void* x, const void* w, void* y, const float* bias, const void* residual, int N, int H, int W,
                     int Cin, int Cout, int act, int num_ctas, cudaStream_t stream, int nextra, const void* const* xe,
                     const void* const* we, float* stats, int* stat_slots);
// Weight-gradient partials into ws: *slices_out slices of dW3 [Cout,3,3,Cin] (then dW1 [Cout,Cin] with dy1), to be added
// by wgrad_reduce_kernel. hb_wgrad_rows_workspace_bytes: the ws bytes wanted (0 = shape not eligible).
int hb_wgrad_rows_try(const void* x, const void* dy, const void* dy1, float* ws, size_t ws_bytes, int N, int H, int W,
                      int Cin, int Cout, int num_ctas, cudaStream_t stream, int* slices_out);
size_t hb_wgrad_rows_workspace_bytes(int N, int H, int W, int Cin, int Cout, int R, int S, int stride, int pad, int dil,
                                     int num_ctas, int has_b1);
