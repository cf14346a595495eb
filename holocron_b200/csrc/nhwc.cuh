// Helpers shared by the kernels over NHWC rows: the pooling kernels (pooling.cu: GlobalMaxPool2d, z_pool, BlurPool2d)
// and the attention kernels (attention.cu: SAM, TripletAttention) take bf16 or fp32 rows and share the max rule, so that
// both route the gradient of a max the same way; the involution and lambda kernels (involution.cu, lambda_layer.cu)
// share the cp.async stager of their shared-memory halo boxes.
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

// ---- bf16 / fp32 rows -----------------------------------------------------------------------
// channels per 16-byte vector of an HB_DTYPE_F32 or HB_DTYPE_BF16 row
inline int vec_width(int dtype) { return dtype == HB_DTYPE_F32 ? 4 : 8; }

// true unless rows of C > 0 logical channels in a pitch of Cp >= C channels, a whole number of 16-byte vectors, hold
// fp32 or bf16
inline bool bad_rows(int C, int Cp, int dtype) {
  return (dtype != HB_DTYPE_F32 && dtype != HB_DTYPE_BF16) || C <= 0 || Cp < C || Cp % vec_width(dtype) != 0;
}

// f(T{}) with T the storage type of dtype, which bad_rows has accepted: f is a generic lambda that names it
// decltype(t)
template <typename F> int with_dtype(int dtype, F&& f) {
  return dtype == HB_DTYPE_F32 ? f(float{}) : f(__nv_bfloat16{});
}

// lanes per row of a kernel that gives each row a group of lanes, one per 16-byte vector: a power of two up to a warp
inline int lane_group(int vectors) { return pow2_at_least(vectors, 32); }

// Xor butterflies over an aligned group of g lanes (a power of two up to 32): every lane of the group ends with the same
// bits. Every lane of the warp must run them, since the shuffles name the full warp.
__device__ __forceinline__ float group_sum(float s, int g) {
  for (int off = 1; off < g; off <<= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  return s;
}

// the max (value mx, index ix, by better()) and the sum sm of the group
__device__ __forceinline__ void group_max_sum(float& mx, int& ix, float& sm, int g) {
  for (int off = 1; off < g; off <<= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, mx, off);
    const int oi = __shfl_xor_sync(0xffffffffu, ix, off);
    sm += __shfl_xor_sync(0xffffffffu, sm, off);
    if (better(om, oi, mx, ix)) {
      mx = om;
      ix = oi;
    }
  }
}

// ---- shared-memory halo boxes ---------------------------------------------------------------
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(valid ? 16 : 0));
}

// Copies the box of bh x bw pixels at (y0, x0) of one image of x [..][H][W][Cp] (bf16), whose first pixel is pix0,
// channel vectors vec0 .. vec0 + nv - 1 of each pixel, into dst [bh][bw][nv] with cp.async: zeros outside the image and
// past the last channel vector. Returns once the box is in shared memory and the CTA has passed a barrier.
__device__ __forceinline__ void stage_box(uint4* dst, const __nv_bfloat16* __restrict__ x, size_t pix0, int H, int W,
                                          int Cp, int y0, int x0, int bh, int bw, int nv, int vec0) {
  const int cv = Cp / 8;
  const int total = bh * bw * nv;
  for (int e = threadIdx.x; e < total; e += blockDim.x) {
    const int v = e % nv, q = e / nv;
    const int hi = y0 + q / bw, wi = x0 + q % bw;
    const bool ok = hi >= 0 && hi < H && wi >= 0 && wi < W && vec0 + v < cv;
    const __nv_bfloat16* src = ok ? x + (pix0 + hi * W + wi) * Cp + (size_t)(vec0 + v) * 8 : x;
    cp_async16(dst + e, src, ok);
  }
  asm volatile("cp.async.commit_group;\n" ::);
  asm volatile("cp.async.wait_group 0;\n" ::);
  __syncthreads();
}

// Opts a kernel into more than the default 48 KiB of dynamic shared memory, raising its ceiling to `limit` bytes (a
// host-side attribute, no synchronisation).
template <typename Kern>
cudaError_t allow_smem(Kern kern, size_t bytes, size_t limit) {
  if (bytes <= 48 * 1024) return cudaSuccess;
  return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)limit);
}

}  // namespace hb
