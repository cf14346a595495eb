// Per-pixel arithmetic of torchvision's colour ops on CUDA tensors (_functional_tensor.py), shared by the batched
// TrivialAugmentWide (autoaugment.cu) and ColorJitter (color_jitter.cu) kernels, the 16-pixel row chunks they read
// and write, and the geometry and reductions of their two launches. Every product and sum is rounded on its own (no
// FMA contraction), as torch runs them as separate kernels.
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

// ---- the two launches of a batch ------------------------------------------------------------------------------------
// A descriptor row (Desc) starts with src, dst, sc, sh, sw, C, H, W: addresses, strides in elements.

// Statistics launch: slice s of `slices` cuts an image's H*W pixels, in row-major order, into runs of
// ceil(H*W / slices) pixels; it is [p0, p1), empty past the end.
struct Slice {
  long long p0, p1;
};

template <typename Desc> __device__ __forceinline__ Slice pixel_slice(const Desc& d, int s, int slices) {
  const long long HW = d.H * d.W, per = (HW + slices - 1) / slices;
  const long long p0 = s * per;
  return {p0, min(HW, p0 + per)};
}

// the address of row-major pixel p of the image's first channel
template <typename T, typename Desc> __device__ __forceinline__ const T* pixel_at(const Desc& d, long long p) {
  const int W = (int)d.W;
  const long long y = p / W, x = p - y * W;
  return reinterpret_cast<const T*>(d.src) + y * d.sh + x * d.sw;
}

// A sum over the CTA in a fixed order, so that floating-point sums repeat bit for bit: a butterfly within each warp,
// then the warp sums in warp order. Every thread gets the result.
template <int kThreads, typename Acc> __device__ __forceinline__ Acc ordered_block_sum(Acc v) {
  __shared__ Acc part[kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
  __syncthreads();
  Acc sum = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) sum += part[w];
  return sum;
}

// Apply launch: CTA n * tiles + t holds tile t of image n, `rows_per_tile` rows of it (one when a row has kThreads
// chunks or more), and a thread takes one kChunk-pixel chunk of a row at a time. False when the grid of N images
// would pass 2^31 - 1 CTAs.
template <int kThreads> inline bool row_tiles(int N, int H, int W, int& rows_per_tile, int& tiles) {
  const int cpr = (W + kChunk - 1) / kChunk;
  rows_per_tile = cpr >= kThreads ? 1 : kThreads / cpr;
  tiles = (H + rows_per_tile - 1) / rows_per_tile;
  return (long long)N * tiles <= 0x7fffffffLL;
}

// The tile of this CTA in image n = blockIdx.x / tiles: rows [y0, y0 + rows), cpr chunks per row.
struct RowTile {
  int y0, rows, cpr;

  __device__ __forceinline__ RowTile(int n, int tiles, int rows_per_tile, int H, int W) {
    const int tile = blockIdx.x - n * tiles;
    y0 = tile * rows_per_tile;
    rows = min(H - y0, rows_per_tile);
    cpr = (W + kChunk - 1) / kChunk;
  }
  __device__ __forceinline__ int items() const { return rows * cpr; }
};

// item i of a tile: row y, first column x0 and len pixels
struct Chunk {
  int y, x0, len;

  __device__ __forceinline__ Chunk(const RowTile& t, int i, int W)
      : y(t.y0 + i / t.cpr), x0((i % t.cpr) * kChunk), len(min(kChunk, W - x0)) {}
};

}  // namespace hb
