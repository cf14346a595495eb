// The tail of the reference's classification chains (references/classification/train.py:100-107, 162-168):
// torchvision's PILToTensor, ConvertImageDtype(torch.float32), Normalize and RandomErasing applied to a batch of images
// of one shape in one launch, reading every pixel of a strided uint8 or fp32 source once and writing a contiguous fp32
// destination once. No host synchronisation: the rows, the fill values, the mean and the std are uploaded by the
// caller from pinned memory.
//
// Image n is one row of the descriptor table, the EraseDesc of hb_erase_batch (row_walk.cuh): the strided source
// [C][H][W], the contiguous fp32 destination [C][H][W], the image's erasing rectangle and its fill. Every element runs
// one op program shared by the batch, in chain order, on an fp32 value that holds the element (a uint8 element as its
// integer value until it is converted):
//   convert    v * f32(1/255): torch's image.to(float32) / 255 on CUDA multiplies by the fp32 reciprocal of the scalar;
//   normalise  (v - mean[c]) / std[c], rounded twice (__fsub_rn, __fdiv_rn): torchvision's sub_ and div_ of device
//              tensors;
//   erase      the element of the rectangle takes its fp32 fill value cast to the dtype current at that point: uint8
//              (before convert) truncates through int64, as torch's copy casts it, fp32 keeps it.
// The walk is erase_kernel's copy mode (row_walk.cuh): a thread owns 16 bytes of a source row, one 16-byte load for a
// uint8 source and four 16-byte stores of its 16 fp32 results (one of each for an fp32 source).
#include "row_walk.cuh"

using namespace hb;

namespace {

constexpr int kThreads = kWalkThreads;

// op codes, packed 8 bits each from the lowest byte up; 0 ends the program
enum TailOp { kEnd = 0, kConvert = 1, kNormalize = 2, kEraseU8 = 3, kEraseF32 = 4 };
constexpr int kMaxOps = 3;

template <typename Ts>
__global__ void __launch_bounds__(kThreads) tail_kernel(const EraseDesc* __restrict__ descs,
                                                        const float* __restrict__ values, int rows, int vpr,
                                                        int blocks_per_image, unsigned ops, int noff) {
  constexpr int V = 16 / sizeof(Ts);
  const int n = blockIdx.x / blocks_per_image;
  const long long item = (long long)(blockIdx.x - n * blocks_per_image) * kThreads + threadIdx.x;
  if (item >= (long long)rows * vpr) return;
  const EraseDesc& d = descs[n];
  const int r = (int)(item / vpr), k = (int)(item - (long long)r * vpr);
  const int C = (int)d.C, H = (int)d.H, W = (int)d.W;
  if (r >= C * H) return;
  const int c = r / H, y = r - c * H;
  const Ts* src_row = reinterpret_cast<const Ts*>(d.src) + c * d.sc + y * d.sh;
  float* dst_row = reinterpret_cast<float*>(d.dst) + ((long long)c * H + y) * W;
  const RowVec<V, float> rv(dst_row, true, k, 0, W);
  if (rv.outside()) return;
  const int xa = rv.xa;
  const long long sw = d.sw;

  const VecN<Ts, V> in = load_vec<Ts, V>(src_row + xa * sw, sw, rv);
  VecN<float, V> out;
#pragma unroll
  for (int j = 0; j < V; ++j) out.v[j] = (float)in.v[j];
  const RectRow rect(d, c, y);
#pragma unroll 1
  for (int i = 0; i < kMaxOps; ++i) {
    const int op = (int)((ops >> (8 * i)) & 0xffu);
    if (op == kEnd) break;
    if (op == kConvert) {
      constexpr float kInv255 = 1.f / 255.f;
#pragma unroll
      for (int j = 0; j < V; ++j) out.v[j] = __fmul_rn(out.v[j], kInv255);
    } else if (op == kNormalize) {
      const float mean = values[noff + c], std = values[noff + C + c];
#pragma unroll
      for (int j = 0; j < V; ++j) out.v[j] = __fdiv_rn(__fsub_rn(out.v[j], mean), std);
    } else if (rect.hit) {
      const bool u8 = op == kEraseU8;
#pragma unroll
      for (int j = 0; j < V; ++j)
        if (rect.covers(xa + j)) {
          const float v = rect.value(values, xa + j);
          out.v[j] = u8 ? (float)cast_fill<uint8_t>(v) : v;
        }
    }
  }
  store_vec<float, V>(dst_row + xa, true, 1, rv, out);
}

template <typename Ts>
int launch(const EraseDesc* descs, const float* values, int N, int rows, int row_len, unsigned ops, int noff,
           cudaStream_t stream) {
  constexpr int V = 16 / sizeof(Ts);
  int vpr, per_image;
  if (!walk_grid(N, rows, row_len, V, vpr, per_image)) return (int)cudaErrorInvalidValue;
  tail_kernel<Ts><<<(unsigned)(N * per_image), kThreads, 0, stream>>>(descs, values, rows, vpr, per_image, ops, noff);
  HB_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" int hb_image_tail_batch(const void* descs, const float* values, int N, int rows, int row_len,
                                   int src_dtype, int ops, int noff, void* stream) {
  if (N <= 0 || rows <= 0 || row_len <= 0 || noff < 0) return (int)cudaErrorInvalidValue;
  for (int i = 0; i < 4; ++i) {
    const int op = (int)(((unsigned)ops >> (8 * i)) & 0xffu);
    if (op > kEraseF32 || (i == kMaxOps && op != kEnd)) return (int)cudaErrorInvalidValue;
  }
  const auto* d = static_cast<const EraseDesc*>(descs);
  auto s = static_cast<cudaStream_t>(stream);
  switch (src_dtype) {
    case HB_DTYPE_F32: return launch<float>(d, values, N, rows, row_len, (unsigned)ops, noff, s);
    case HB_DTYPE_U8: return launch<uint8_t>(d, values, N, rows, row_len, (unsigned)ops, noff, s);
    default: return (int)cudaErrorInvalidValue;
  }
}
