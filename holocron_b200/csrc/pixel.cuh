// Per-pixel arithmetic of torchvision's colour ops on CUDA tensors (_functional_tensor.py), shared by the batched
// TrivialAugmentWide (autoaugment.cu) and ColorJitter (color_jitter.cu) kernels, and the 16-pixel row chunks they read
// and write. Every product and sum is rounded on its own (no FMA contraction), as torch runs them as separate kernels.
#pragma once
#include "common.cuh"

namespace hb {

constexpr int kChunk = 16;  // pixels of one row a thread owns

// uint8 images: torch's float -> uint8 cast of a value clamped to [0, 255] truncates
__device__ __forceinline__ uint8_t trunc_u8(float v) { return (uint8_t)__float2int_rz(clamp_nan(v, 0.f, 255.f)); }

// _blend of a uint8 image: trunc(clamp(f32(r)*v + f32(1 - r)*b, 0, 255))
__device__ __forceinline__ uint8_t blend(float r, float q, uint8_t v, float b) {
  return trunc_u8(__fadd_rn(__fmul_rn(r, (float)v), __fmul_rn(q, b)));
}

// rgb_to_grayscale of a uint8 image: trunc((0.2989*r + 0.587*g) + 0.114*b)
__device__ __forceinline__ uint8_t gray(uint8_t r, uint8_t g, uint8_t b) {
  return (uint8_t)__float2int_rz(
      __fadd_rn(__fadd_rn(__fmul_rn(0.2989f, (float)r), __fmul_rn(0.587f, (float)g)), __fmul_rn(0.114f, (float)b)));
}

__device__ __forceinline__ Vec16<uint8_t> load_chunk(const uint8_t* p, long long sw, int len) {
  Vec16<uint8_t> v;
  if (len == kChunk && sw == 1 && aligned16(p)) return ld16(p);
  v.raw = make_uint4(0, 0, 0, 0);
#pragma unroll
  for (int j = 0; j < kChunk; ++j)
    if (j < len) v.v[j] = p[j * sw];
  return v;
}

__device__ __forceinline__ void store_chunk(uint8_t* p, const Vec16<uint8_t>& v, int len) {
  if (len == kChunk && aligned16(p)) {
    st16(p, v);
    return;
  }
#pragma unroll
  for (int j = 0; j < kChunk; ++j)
    if (j < len) p[j] = v.v[j];
}

// ---- fp32 counterparts ----------------------------------------------------------------------------------------------

// _blend of an fp32 image: clamp(f32(r)*v + f32(1 - r)*b, 0, 1), no cast
__device__ __forceinline__ float blend_f32(float r, float q, float v, float b) {
  return clamp_nan(__fadd_rn(__fmul_rn(r, v), __fmul_rn(q, b)), 0.f, 1.f);
}

// rgb_to_grayscale of an fp32 image: (0.2989*r + 0.587*g) + 0.114*b
__device__ __forceinline__ float gray_f32(float r, float g, float b) {
  return __fadd_rn(__fadd_rn(__fmul_rn(0.2989f, r), __fmul_rn(0.587f, g)), __fmul_rn(0.114f, b));
}

// One 16-byte vector of an fp32 row holds 4 pixels: the first min(len, 4) pixels from p, column stride sw.
__device__ __forceinline__ Vec16<float> load_chunk(const float* p, long long sw, int len) {
  Vec16<float> v;
  if (len >= Vec16<float>::N && sw == 1 && aligned16(p)) return ld16(p);
  v.raw = make_uint4(0, 0, 0, 0);
#pragma unroll
  for (int j = 0; j < Vec16<float>::N; ++j)
    if (j < len) v.v[j] = p[j * sw];
  return v;
}

__device__ __forceinline__ void store_chunk(float* p, const Vec16<float>& v, int len) {
  if (len >= Vec16<float>::N && aligned16(p)) {
    st16(p, v);
    return;
  }
#pragma unroll
  for (int j = 0; j < Vec16<float>::N; ++j)
    if (j < len) p[j] = v.v[j];
}

}  // namespace hb
