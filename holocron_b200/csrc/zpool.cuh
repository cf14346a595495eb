// Max / mean reduction helpers shared by the pooling kernels (pooling.cu: GlobalMaxPool2d, z_pool) and the attention
// kernels (attention.cu: the Z-pooled planes of TripletAttention), so that both route the gradient of a max the same way.
#pragma once
#include "common.cuh"

namespace hb {

// (v, i) replaces (cur, ci): NaN first (the lowest-index NaN), then the larger value, then the lower index, which is the
// element torch's max(dim).indices names. The state (-inf, kNoIndex) loses to every element, -inf included. The order is
// total, so any fixed combination tree gives the same winner.
__device__ __forceinline__ bool better(float v, int i, float cur, int ci) {
  if (cur != cur) return v != v && i < ci;
  if (v != v || v > cur) return true;
  return v == cur && i < ci;
}

constexpr int kNoIndex = 0x7fffffff;

// fp32 -> T for a value that was read from a T: the bits come back unchanged (a NaN keeps its sign and payload, which
// a rounding conversion would replace by the canonical NaN)
template <typename T> __device__ __forceinline__ T same_bits(float f);
template <> __device__ __forceinline__ float same_bits<float>(float f) { return f; }
template <> __device__ __forceinline__ __nv_bfloat16 same_bits<__nv_bfloat16>(float f) {
  return __ushort_as_bfloat16((unsigned short)(__float_as_uint(f) >> 16));
}

// V fp32 values -> one vector of T, lanes c0 + l >= C written as zeros; kExact for values read from a T (the max)
template <typename T, bool kExact = false>
__device__ __forceinline__ Vec16<T> pack(const float* f, int c0, int C) {
  Vec16<T> v;
#pragma unroll
  for (int l = 0; l < Vec16<T>::N; ++l) {
    const float x = c0 + l < C ? f[l] : 0.f;
    v.v[l] = kExact ? same_bits<T>(x) : from_f<T>(x);
  }
  return v;
}

// the smallest power of two >= v, capped at cap
inline int pow2_at_least(int v, int cap) {
  int g = 1;
  while (g < v && g < cap) g <<= 1;
  return g;
}

}  // namespace hb
