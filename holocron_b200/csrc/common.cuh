// Shared device helpers for the holocron_b200 sm_90a kernels.
// Everything here is header-only; each .cu translation unit includes it.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#define HB_DTYPE_F32 0
#define HB_DTYPE_BF16 1
#define HB_DTYPE_F16 2
#define HB_DTYPE_U8 3
#define HB_DTYPE_F64 4


#define HB_NUM_SMS (hb::num_sms())

#include <atomic>
extern std::atomic<long long> g_hb_launches;  // defined in runtime.cu

// after every kernel launch: count it and surface launch-configuration errors as the return code
#define HB_LAUNCH_CHECK()                          \
  do {                                             \
    g_hb_launches.fetch_add(1, std::memory_order_relaxed); \
    cudaError_t e__ = cudaGetLastError();          \
    if (e__ != cudaSuccess) return (int)e__;       \
  } while (0)

namespace hb {

// SM count of the current device (H100 SXM: 132, H100 PCIe: 114): sizes the persistent grids and the partial-sum slot
// counts. Read from the runtime once per device.
inline int num_sms() {
  static int cache[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cache[dev] == 0) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
    cache[dev] = v;
  }
  return cache[dev];
}

// ---- scalar conversions -------------------------------------------------------------------
template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }

template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }

// ---- 128-bit vector container -------------------------------------------------------------
template <typename T> struct Vec16 {
  static constexpr int N = 16 / sizeof(T);
  union { uint4 raw; T v[N]; };
};

template <typename T> __device__ __forceinline__ Vec16<T> ld16(const T* p) {
  Vec16<T> r; r.raw = *reinterpret_cast<const uint4*>(p); return r;
}
// streaming (read-once) 128-bit load that does not allocate in L1 (coherent path: safe for in-place ops)
template <typename T> __device__ __forceinline__ Vec16<T> ld16_stream(const T* p) {
  Vec16<T> r;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.raw.x), "=r"(r.raw.y), "=r"(r.raw.z), "=r"(r.raw.w) : "l"(p));
  return r;
}
template <typename T> __device__ __forceinline__ void st16(T* p, const Vec16<T>& v) {
  *reinterpret_cast<uint4*>(p) = v.raw;
}

// 8 bf16 <-> 8 fp32. There is deliberately no load8: each caller picks its cache hint (unpack8(ld16_stream(p), f) for
// read-once streams, unpack8(ld16(p), f) for data neighbouring threads re-read through L1).
__device__ __forceinline__ void unpack8(const Vec16<__nv_bfloat16>& v, float* f) {
#pragma unroll
  for (int j = 0; j < 8; ++j) f[j] = __bfloat162float(v.v[j]);
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float* f) {
  Vec16<__nv_bfloat16> v;
#pragma unroll
  for (int j = 0; j < 8; ++j) v.v[j] = __float2bfloat16_rn(f[j]);
  st16(p, v);
}

__host__ __device__ __forceinline__ bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// ---- NaN-propagating clamps -------------------------------------------------------------
// torch.relu / clamp / max propagate NaN; CUDA's fmaxf / fminf return the non-NaN operand, which would silently launder a NaN
// activation into 0 at the first ReLU - and with it the reference trainer's NaN-loss detection (trainer/core.py:153-159).
__device__ __forceinline__ float relu_nan(float z) { return z < 0.f ? 0.f : z; }
__device__ __forceinline__ float clamp_nan(float z, float lo, float hi) { return z < lo ? lo : (z > hi ? hi : z); }
__device__ __forceinline__ float max_nan(float a, float b) { return (a > b || a != a) ? a : b; }

// ---- reductions ---------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide sum; result valid in thread 0 (and broadcast to all when kBroadcast).
// `scratch` must hold >= 32 elements of T in shared memory.
template <typename T, bool kBroadcast = false>
__device__ __forceinline__ T block_sum(T v, T* scratch) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nwarps = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();  // protect scratch reuse across consecutive calls
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  if (warp == 0) {
    T t = lane < nwarps ? scratch[lane] : T(0);
    t = warp_sum(t);
    if (lane == 0) scratch[0] = t;
  }
  if (kBroadcast) { __syncthreads(); return scratch[0]; }
  return (threadIdx.x == 0) ? scratch[0] : T(0);
}

// grid sizing for streaming passes: enough CTAs for >= 2 waves but capped at a multiple of the SM count
__host__ inline int stream_grid(size_t work_items, int per_block, int max_waves = 8) {
  size_t need = (work_items + per_block - 1) / per_block;
  size_t cap = (size_t)HB_NUM_SMS * max_waves;
  if (need < 1) need = 1;
  return (int)(need < cap ? need : cap);
}

// Output extent of a window of k taps (dilation dil) sliding with `stride` over `in` pixels padded by `pad` on both
// sides. False unless in, k, stride, dil >= 1, pad >= 0, the dilated window fits the padded input and the extent fits
// an int. The span is computed in 64 bits and tested before the division, which truncates towards zero: on its own,
// (in + 2 * pad - dil * (k - 1) - 1) / stride + 1 gives 1 for a window up to stride - 1 pixels too large.
inline bool window_out(int in, int k, int stride, int pad, int dil, int& out) {
  if (in < 1 || k < 1 || stride < 1 || dil < 1 || pad < 0) return false;
  const long long span = (long long)in + 2LL * pad - (long long)dil * (k - 1) - 1;
  if (span < 0 || span / stride >= 0x7fffffffLL) return false;
  out = (int)(span / stride + 1);
  return true;
}

template <typename T> struct Type { using type = T; };

// f(Type<T>{}) for the dtype code; cudaErrorInvalidValue for an unknown code
template <class F>
int dispatch_dtype(int dtype, F f) {
  switch (dtype) {
    case HB_DTYPE_F32: return f(Type<float>{});
    case HB_DTYPE_BF16: return f(Type<__nv_bfloat16>{});
    case HB_DTYPE_F16: return f(Type<__half>{});
    default: return (int)cudaErrorInvalidValue;
  }
}

}  // namespace hb
