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
// is contiguous and aligned too. Other elements go one at a time (the walk of row_walk.cuh). No atomics, no shared
// memory.
#include "row_walk.cuh"

using namespace hb;

namespace {

constexpr int kThreads = kWalkThreads;

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
  const RowVec<V, T> rv(dst_row + x0, dst_contig, k, x0, len);
  if (rv.outside()) return;
  const int xa = rv.xa;

  VecN<T, V> out;
  if (!in_place) out = load_vec<T, V>(src_row + xa * sw, sw, rv);
  const RectRow rect(d, c, y);
  if (rect.hit) {
#pragma unroll
    for (int j = 0; j < V; ++j)
      if (rect.covers(xa + j)) out.v[j] = cast_fill<T>(rect.value(values, xa + j));
  }
  store_vec<T, V>(dst_row + xa * (dst_contig ? 1 : sw), dst_contig, sw, rv, out);
}

template <typename T>
int launch(const EraseDesc* descs, const float* values, int N, int rows, int row_len, cudaStream_t stream) {
  constexpr int V = 16 / sizeof(T);
  int vpr, per_image;
  if (!walk_grid(N, rows, row_len, V, vpr, per_image)) return (int)cudaErrorInvalidValue;
  erase_kernel<T><<<(unsigned)(N * per_image), kThreads, 0, stream>>>(descs, values, rows, vpr, per_image);
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
