// Batched random erasing (torchvision.transforms.RandomErasing.forward / get_params, the training transform of the
// reference's classification recipe), one launch per batch of images of one shape.
//
// Image n is described by one row of a device table (EraseDesc, uploaded by the caller from pinned memory together
// with the fp32 value buffer, without a host synchronisation): a strided source [C][H][W] read in place, a destination,
// the rectangle (top, left, h, w) and its fill. Two modes, chosen per row:
//   copy      dst != src: dst is contiguous [C][H][W]; every pixel is written, the source's outside the rectangle and
//             the fill inside it (torchvision's img.clone() then img[..., i:i+h, j:j+w] = v).
//   in place  dst == src: only the rectangle is written, through the source's strides (inplace=True).
// Fills: 0 none (the rectangle is empty: get_params found none in its 10 attempts and torchvision assigns the image to
// itself), 1 one value per channel at values[voff + c], 2 one value per pixel at values[voff + (c*h + y)*w + x] (the
// host's torch.empty([C, h, w]).normal_() draw for value="random"). The fp32 values are cast to the image dtype as
// torch's copy casts them: fp16 / bf16 round to nearest even, uint8 truncates toward zero through int64 and keeps the
// low byte (c10's static_cast_with_inter_type), fp64 widens exactly.
//
// A thread owns one 16-byte vector of a destination row segment (the whole row in copy mode, the rectangle's columns
// in place). Vectors are aligned to 16 bytes in memory: the first one of a row starts up to V - 1 elements early and
// covers its valid elements only, so every full vector is one 128-bit store, and one 128-bit load where the source row
// is contiguous and aligned too. Other elements go one at a time. No atomics, no shared memory.
#include "common.cuh"

using namespace hb;

namespace {

constexpr int kThreads = 256;

enum Fill { kNone = 0, kPerChannel = 1, kPerPixel = 2 };

// One row of the descriptor table (16 x int64, include/holocron_b200.h). Pointers are addresses, strides count
// elements of the image dtype.
struct EraseDesc {
  long long src, dst, sc, sh, sw;
  long long C, H, W, top, left, h, w, fill, voff, reserved0, reserved1;
};

template <typename T> __device__ __forceinline__ T cast_fill(float v);
template <> __device__ __forceinline__ float cast_fill<float>(float v) { return v; }
template <> __device__ __forceinline__ double cast_fill<double>(float v) { return (double)v; }
template <> __device__ __forceinline__ __half cast_fill<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 cast_fill<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ uint8_t cast_fill<uint8_t>(float v) {
  return static_cast<uint8_t>(static_cast<long long>(v));
}

// One CTA per (image, 256 vectors of its rows). rows: the most row segments an image has (C*H in copy mode, C*h in
// place); vpr: vectors per row segment, one more than the longest segment needs, for the alignment head.
template <typename T>
__global__ void __launch_bounds__(kThreads) erase_kernel(const EraseDesc* __restrict__ descs,
                                                         const float* __restrict__ values, int rows, int vpr,
                                                         int blocks_per_image) {
  constexpr int V = 16 / sizeof(T);
  const int n = blockIdx.x / blocks_per_image;
  const long long item = (long long)(blockIdx.x - n * blocks_per_image) * kThreads + threadIdx.x;
  if (item >= (long long)rows * vpr) return;
  const EraseDesc& d = descs[n];
  const int r = (int)(item / vpr), k = (int)(item - (long long)r * vpr);
  const int H = (int)d.H, W = (int)d.W, top = (int)d.top, left = (int)d.left, h = (int)d.h, w = (int)d.w;
  const int fill = (int)d.fill;
  const bool in_place = d.dst == d.src;
  if (in_place && (fill == kNone || r >= (int)d.C * h)) return;
  if (!in_place && r >= (int)d.C * H) return;

  int c, y, x0, len;
  if (in_place) {
    c = r / h;
    y = top + (r - c * h);
    x0 = left;
    len = w;
  } else {
    c = r / H;
    y = r - c * H;
    x0 = 0;
    len = W;
  }
  const T* src_row = reinterpret_cast<const T*>(d.src) + c * d.sc + y * d.sh;
  const long long sw = d.sw;
  // destination element x of this row: contiguous in copy mode, the source's strides in place
  T* dst_row = in_place ? reinterpret_cast<T*>(d.dst) + c * d.sc + y * d.sh
                        : reinterpret_cast<T*>(d.dst) + ((long long)c * H + y) * W;
  const bool dst_contig = !in_place || sw == 1;
  const int head = dst_contig ? (int)((reinterpret_cast<uintptr_t>(dst_row + x0) & 15) / sizeof(T)) : 0;
  const int e0 = k * V - head;  // element offset of this vector within the row segment
  if (e0 >= len) return;
  const int xa = x0 + e0;  // column of the vector's first element
  const bool full = e0 >= 0 && e0 + V <= len;

  const bool row_in_rect = fill != kNone && y >= top && y < top + h;
  // value of column xx of this row: values[vrow + xx] per pixel, values[vrow] per channel
  const long long vrow = d.voff + (fill == kPerPixel ? ((long long)c * h + (y - top)) * w - left : c);

  Vec16<T> out;
  if (!in_place) {
    const T* s = src_row + xa * sw;
    if (full && sw == 1 && aligned16(s)) {
      out = ld16(s);
    } else {
#pragma unroll
      for (int j = 0; j < V; ++j)
        if (e0 + j >= 0 && e0 + j < len) out.v[j] = s[j * sw];
    }
  }
  if (row_in_rect) {
#pragma unroll
    for (int j = 0; j < V; ++j) {
      const int xx = xa + j;
      if (xx >= left && xx < left + w) out.v[j] = cast_fill<T>(values[fill == kPerPixel ? vrow + xx : vrow]);
    }
  }
  T* o = dst_row + xa * (dst_contig ? 1 : sw);
  if (full && dst_contig) {
    st16(o, out);
  } else {
#pragma unroll
    for (int j = 0; j < V; ++j)
      if (e0 + j >= 0 && e0 + j < len) o[j * (dst_contig ? 1 : sw)] = out.v[j];
  }
}

template <typename T>
int launch(const EraseDesc* descs, const float* values, int N, int rows, int row_len, cudaStream_t stream) {
  constexpr int V = 16 / sizeof(T);
  const int vpr = (row_len + V - 1) / V + 1;
  const long long per_image = ((long long)rows * vpr + kThreads - 1) / kThreads;
  if (per_image > 0x7fffffffLL || (long long)N * per_image > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
  erase_kernel<T><<<(unsigned)(N * per_image), kThreads, 0, stream>>>(descs, values, rows, vpr, (int)per_image);
  HB_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" int hb_erase_batch(const void* descs, const float* values, int N, int rows, int row_len, int dtype,
                              void* stream) {
  if (N <= 0 || rows < 0 || row_len < 0) return (int)cudaErrorInvalidValue;
  // an in-place batch without a rectangle writes nothing; its launch still happens and returns at once
  rows = rows > 0 ? rows : 1;
  row_len = row_len > 0 ? row_len : 1;
  const auto* d = static_cast<const EraseDesc*>(descs);
  auto s = static_cast<cudaStream_t>(stream);
  switch (dtype) {
    case HB_DTYPE_F32: return launch<float>(d, values, N, rows, row_len, s);
    case HB_DTYPE_BF16: return launch<__nv_bfloat16>(d, values, N, rows, row_len, s);
    case HB_DTYPE_F16: return launch<__half>(d, values, N, rows, row_len, s);
    case HB_DTYPE_U8: return launch<uint8_t>(d, values, N, rows, row_len, s);
    case HB_DTYPE_F64: return launch<double>(d, values, N, rows, row_len, s);
    default: return (int)cudaErrorInvalidValue;
  }
}
