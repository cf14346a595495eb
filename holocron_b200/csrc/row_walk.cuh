// The row-segment walk shared by the batched erasing (erase.cu) and image-tail (image_tail.cu) kernels: the
// descriptor row of an image and its rectangle, the thread-to-vector mapping of a destination row segment, the
// vector loads and stores, and the cast of a fill value to the image dtype.
//
// A thread owns one vector of V source elements of a row segment. Vectors are aligned in the destination: the first
// one of a row starts up to V - 1 elements early, so that its destination elements start on a V * sizeof(Td)-byte
// boundary, and covers its valid elements only. Every full vector is then whole 128-bit stores, and one 128-bit load
// where the source row is contiguous and aligned too. Other elements go one at a time.
#pragma once
#include "common.cuh"

namespace hb {

constexpr int kWalkThreads = 256;

// fills of a rectangle: 0 none (nothing erased), 1 one value per channel at values[voff + c], 2 one value per pixel at
// values[voff + (c*h + y)*w + x]
enum Fill { kNone = 0, kPerChannel = 1, kPerPixel = 2 };

// One row of the descriptor table (16 x int64, include/holocron_b200.h). Pointers are addresses, strides count
// elements of the source dtype.
struct EraseDesc {
  long long src, dst, sc, sh, sw;
  long long C, H, W, top, left, h, w, fill, voff, reserved0, reserved1;
};

// The fp32 fill value cast to the image dtype as torch's copy casts it: fp16 / bf16 round to nearest even, uint8
// truncates toward zero through int64 and keeps the low byte (c10's static_cast_with_inter_type), fp64 widens exactly.
template <typename T> __device__ __forceinline__ T cast_fill(float v);
template <> __device__ __forceinline__ float cast_fill<float>(float v) { return v; }
template <> __device__ __forceinline__ double cast_fill<double>(float v) { return (double)v; }
template <> __device__ __forceinline__ __half cast_fill<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 cast_fill<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ uint8_t cast_fill<uint8_t>(float v) {
  return static_cast<uint8_t>(static_cast<long long>(v));
}

// V elements of T in whole 16-byte words
template <typename T, int V> struct VecN {
  static constexpr int kWords = V * (int)sizeof(T) / 16;
  union { uint4 raw[kWords]; T v[V]; };
};

// Thread k's vector of a row segment of len elements from column x0, V source elements to a vector; dst_x0 is the
// destination of the segment's first element.
template <int V, typename Td> struct RowVec {
  int e0;     // element offset of the vector within the segment (negative in the alignment head)
  int xa;     // column of the vector's first element
  int len;
  bool full;  // all V elements lie in the segment

  __device__ __forceinline__ RowVec(const Td* dst_x0, bool dst_contig, int k, int x0, int len_) : len(len_) {
    const int head =
        dst_contig ? (int)((reinterpret_cast<uintptr_t>(dst_x0) & (V * sizeof(Td) - 1)) / sizeof(Td)) : 0;
    e0 = k * V - head;
    xa = x0 + e0;
    full = e0 >= 0 && e0 + V <= len;
  }
  __device__ __forceinline__ bool outside() const { return e0 >= len; }
  __device__ __forceinline__ bool valid(int j) const { return e0 + j >= 0 && e0 + j < len; }
};

// The vector's source elements from s (its first column), column stride sw
template <typename Ts, int V, typename Td>
__device__ __forceinline__ VecN<Ts, V> load_vec(const Ts* s, long long sw, const RowVec<V, Td>& rv) {
  VecN<Ts, V> out;
  if (rv.full && sw == 1 && aligned16(s)) {
#pragma unroll
    for (int q = 0; q < VecN<Ts, V>::kWords; ++q) out.raw[q] = reinterpret_cast<const uint4*>(s)[q];
  } else {
#pragma unroll
    for (int j = 0; j < V; ++j)
      if (rv.valid(j)) out.v[j] = s[j * sw];
  }
  return out;
}

// The vector's destination elements to o (its first column), column stride 1 when contig, else sw
template <typename Td, int V>
__device__ __forceinline__ void store_vec(Td* o, bool contig, long long sw, const RowVec<V, Td>& rv,
                                          const VecN<Td, V>& out) {
  if (rv.full && contig) {
#pragma unroll
    for (int q = 0; q < VecN<Td, V>::kWords; ++q) reinterpret_cast<uint4*>(o)[q] = out.raw[q];
  } else {
#pragma unroll
    for (int j = 0; j < V; ++j)
      if (rv.valid(j)) o[j * (contig ? 1 : sw)] = out.v[j];
  }
}

// Row y of channel c as it meets the image's rectangle: which columns it covers and their fp32 fill values
struct RectRow {
  bool hit;
  bool per_pixel;
  int left, w;
  long long vrow;  // values[vrow + x] per pixel, values[vrow] per channel

  __device__ __forceinline__ RectRow(const EraseDesc& d, int c, int y) {
    const int top = (int)d.top, h = (int)d.h, fill = (int)d.fill;
    left = (int)d.left;
    w = (int)d.w;
    hit = fill != kNone && y >= top && y < top + h;
    per_pixel = fill == kPerPixel;
    vrow = d.voff + (per_pixel ? ((long long)c * h + (y - top)) * w - left : c);
  }
  __device__ __forceinline__ bool covers(int x) const { return x >= left && x < left + w; }
  __device__ __forceinline__ float value(const float* values, int x) const {
    return values[per_pixel ? vrow + x : vrow];
  }
};

// Grid of a walk over N images of `rows` row segments of at most row_len elements, V to a vector: vpr vectors per
// segment (one more than the longest needs, for the alignment head) and per_image CTAs per image. False when the grid
// would pass 2^31 - 1 CTAs.
inline bool walk_grid(int N, int rows, int row_len, int V, int& vpr, int& per_image) {
  vpr = (row_len + V - 1) / V + 1;
  const long long per = ((long long)rows * vpr + kWalkThreads - 1) / kWalkThreads;
  if (per > 0x7fffffffLL || (long long)N * per > 0x7fffffffLL) return false;
  per_image = (int)per;
  return true;
}

}  // namespace hb
