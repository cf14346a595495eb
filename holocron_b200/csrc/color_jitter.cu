// Batched ColorJitter (torchvision.transforms.ColorJitter.forward: adjust_brightness, adjust_contrast,
// adjust_saturation and adjust_hue in a drawn order, as the reference's segmentation and detection recipes apply it,
// references/segmentation/train.py:133-140, references/detection/train.py:116-125) on uint8 or fp32 images of one
// shape: at most two launches per batch and no host synchronisation.
//
// Image n is one row of a device table (JitterDesc, uploaded by the caller from pinned memory together with the fp32
// parameters and the list of images with a contrast factor): a strided source [C][H][W] read in place, a contiguous
// destination [C][H][W], the image's ops in their drawn order and their parameters. Every op is a function of a
// pixel's channels, except the contrast mean, which is a sum over the image of the grayscale of what the ops drawn
// before contrast made of it. The arithmetic is torchvision's tensor path on CUDA (_functional_tensor.py), fp32
// operation by fp32 operation, with no contraction into FMAs where torch runs the products and the sums as separate
// kernels:
//   brightness, contrast, saturation: _blend, b = 0, the grayscale mean, the pixel's grayscale (pixel.cuh);
//   hue: convert_image_dtype to fp32 (uint8: v * f32(1/255), torch's division by a scalar), _rgb2hsv (true divisions),
//       (h + f) % 1 (torch's remainder), _hsv2rgb (its einsum multiplies by a one-hot mask: it picks one term), and
//       convert_image_dtype back (uint8: trunc(x * f32(255.999))).
// A uint8 image is rounded to uint8 after every op, as every torchvision op returns uint8; an fp32 one is clamped to
// [0, 1] after every blend. Saturation and hue leave a one-channel image unchanged.
//
// Launch 1 (only when an image has a contrast factor): one CTA per (image with contrast, pixel slice) applies the
// image's ops before contrast to each pixel of its slice and sums the grayscale (uint8: truncated to uint8; one
// channel: the pixel) into scratch[k][slice]: an exact int64 sum for uint8, an fp64 sum in a fixed order for fp32. No
// global atomics and no memset.
// Launch 2: one CTA per (image, tile of rows); a thread owns a 16-pixel chunk of one row for every channel, read and
// written with 16-byte vectors where rows are contiguous and aligned. Where the image has a contrast op, every thread
// sums its slice partials in slice order and forms the mean as torch's CUDA mean does (the fp32 sum times the fp32
// factor outputs / inputs: 1 / (H*W) for one image); then the image's whole chain runs in registers. Both launches
// run the chain with one device function, run_ops: launch 1 recomputes the ops before contrast rather than storing an
// intermediate image.
#include <type_traits>

#include "pixel.cuh"

using namespace hb;

namespace {

constexpr int kThreads = 256;

// op codes: torchvision's fn_idx values
enum Op { kBrightness = 0, kContrast = 1, kSaturation = 2, kHue = 3 };
// fp32 parameters of one image (8 floats): r and 1 - r of each blend at 2 * op and 2 * op + 1, the hue factor, the
// factor of the contrast mean
constexpr int kParams = 8;
constexpr int kHueFactor = 6;
constexpr int kMeanFactor = 7;

// One row of the descriptor table (16 x int64, include/holocron_b200.h). Pointers are addresses, strides count
// elements.
struct JitterDesc {
  long long src, dst, sc, sh, sw, C, H, W, n_ops, op[4], contrast_at, stat, reserved;
};

// An image's chain as a thread holds it: op codes packed 8 bits each (so a runtime op index needs no local array).
struct Chain {
  unsigned ops;
  int n, at;
  bool rgb;
  float p[kParams];
  __device__ __forceinline__ int op(int i) const { return (int)((ops >> (8 * i)) & 0xffu); }
};

__device__ __forceinline__ Chain load_chain(const JitterDesc& d, const float* P) {
  Chain ch;
  ch.ops = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (i < d.n_ops) ch.ops |= (unsigned)(d.op[i] & 0xff) << (8 * i);
  ch.n = (int)d.n_ops;
  ch.at = (int)d.contrast_at;
  ch.rgb = d.C == 3;
#pragma unroll
  for (int i = 0; i < kParams; ++i) ch.p[i] = P[i];
  return ch;
}

__device__ __forceinline__ float min_nan(float a, float b) { return (a < b || a != a) ? a : b; }

// torch.remainder(x, 1.0) on CUDA: fmod, moved into [0, 1) when negative (the sum can round up to 1)
__device__ __forceinline__ float remainder1(float x) {
  float m = fmodf(x, 1.f);
  if (m != 0.f && m < 0.f) m = __fadd_rn(m, 1.f);
  return m;
}

// adjust_hue of one fp32 RGB pixel in [0, 1] (after convert_image_dtype)
__device__ __forceinline__ void hue_f32(float f, float& r, float& g, float& b) {
  // _rgb2hsv
  const float maxc = max_nan(max_nan(r, g), b), minc = min_nan(min_nan(r, g), b);
  const bool eqc = maxc == minc;
  const float cr = __fsub_rn(maxc, minc);
  const float s = __fdiv_rn(cr, eqc ? 1.f : maxc);
  const float div = eqc ? 1.f : cr;
  const float rc = __fdiv_rn(__fsub_rn(maxc, r), div), gc = __fdiv_rn(__fsub_rn(maxc, g), div),
              bc = __fdiv_rn(__fsub_rn(maxc, b), div);
  // boolean masks times values: 0 * x keeps the sign of zero torch gives
  const float hr = __fmul_rn(maxc == r ? 1.f : 0.f, __fsub_rn(bc, gc));
  const float hg = __fmul_rn(maxc == g && maxc != r ? 1.f : 0.f, __fsub_rn(__fadd_rn(2.f, rc), bc));
  const float hb = __fmul_rn(maxc != g && maxc != r ? 1.f : 0.f, __fsub_rn(__fadd_rn(4.f, gc), rc));
  float h = __fadd_rn(__fadd_rn(hr, hg), hb);
  h = fmodf(__fadd_rn(__fmul_rn(h, 1.f / 6.f), 1.f), 1.f);  // h / 6.0: torch multiplies by the fp32 reciprocal
  h = remainder1(__fadd_rn(h, f));
  // _hsv2rgb
  const float v = maxc;
  const float h6 = __fmul_rn(h, 6.f), fi = floorf(h6), fr = __fsub_rn(h6, fi);
  const float p = clamp_nan(__fmul_rn(v, __fsub_rn(1.f, s)), 0.f, 1.f);
  const float q = clamp_nan(__fmul_rn(v, __fsub_rn(1.f, __fmul_rn(s, fr))), 0.f, 1.f);
  const float t = clamp_nan(__fmul_rn(v, __fsub_rn(1.f, __fmul_rn(s, __fsub_rn(1.f, fr)))), 0.f, 1.f);
  int i = (int)fi % 6;
  if (i < 0) i += 6;
  switch (i) {
    case 0: r = v, g = t, b = p; break;
    case 1: r = q, g = v, b = p; break;
    case 2: r = p, g = v, b = t; break;
    case 3: r = p, g = q, b = v; break;
    case 4: r = t, g = p, b = v; break;
    default: r = v, g = p, b = q; break;
  }
}

// Pixels of either dtype travel as fp32 (a uint8 pixel as its integer value).
template <bool kU8> __device__ __forceinline__ float blend_px(float r, float q, float v, float b) {
  if (kU8) return (float)blend(r, q, (uint8_t)v, b);
  return blend_f32(r, q, v, b);
}

template <bool kU8> __device__ __forceinline__ float gray_px(float r, float g, float b) {
  if (kU8) return (float)gray((uint8_t)r, (uint8_t)g, (uint8_t)b);
  return gray_f32(r, g, b);
}

template <bool kU8> __device__ __forceinline__ void hue_px(float f, float& r, float& g, float& b) {
  if (!kU8) {
    hue_f32(f, r, g, b);
    return;
  }
  constexpr float kInv255 = 1.f / 255.f;
  float x = __fmul_rn(r, kInv255), y = __fmul_rn(g, kInv255), z = __fmul_rn(b, kInv255);
  hue_f32(f, x, y, z);
  // convert_image_dtype(fp32 -> uint8): trunc(x * 255.999)
  r = (float)__float2int_rz(__fmul_rn(x, 255.999f));
  g = (float)__float2int_rz(__fmul_rn(y, 255.999f));
  b = (float)__float2int_rz(__fmul_rn(z, 255.999f));
}

// Applies ops [from, to) of the chain to kPix pixels (channels r, g, b; a one-channel image uses r alone). mean: the
// contrast mean, read only when contrast is in the range.
template <bool kU8, int kPix>
__device__ __forceinline__ void run_ops(const Chain& ch, int from, int to, float mean, float (&r)[kPix],
                                        float (&g)[kPix], float (&b)[kPix]) {
  for (int i = from; i < to; ++i) {
    const int op = ch.op(i);
    if (op == kBrightness || op == kContrast) {
      const bool c = op == kContrast;
      const float pr = c ? ch.p[2 * kContrast] : ch.p[2 * kBrightness],
                  pq = c ? ch.p[2 * kContrast + 1] : ch.p[2 * kBrightness + 1], base = c ? mean : 0.f;
#pragma unroll
      for (int j = 0; j < kPix; ++j) {
        r[j] = blend_px<kU8>(pr, pq, r[j], base);
        if (ch.rgb) g[j] = blend_px<kU8>(pr, pq, g[j], base), b[j] = blend_px<kU8>(pr, pq, b[j], base);
      }
    } else if (op == kSaturation && ch.rgb) {
      const float pr = ch.p[2 * kSaturation], pq = ch.p[2 * kSaturation + 1];
#pragma unroll
      for (int j = 0; j < kPix; ++j) {
        const float l = gray_px<kU8>(r[j], g[j], b[j]);
        r[j] = blend_px<kU8>(pr, pq, r[j], l);
        g[j] = blend_px<kU8>(pr, pq, g[j], l);
        b[j] = blend_px<kU8>(pr, pq, b[j], l);
      }
    } else if (op == kHue && ch.rgb) {
#pragma unroll
      for (int j = 0; j < kPix; ++j) hue_px<kU8>(ch.p[kHueFactor], r[j], g[j], b[j]);
    }
  }
}

template <typename T>
__device__ __forceinline__ void stats_body(const JitterDesc* __restrict__ descs, const float* __restrict__ params,
                                           const long long* __restrict__ stat_images, void* scratch, int slices) {
  constexpr bool kU8 = sizeof(T) == 1;
  using Acc = typename std::conditional<kU8, long long, double>::type;
  const int s = blockIdx.x % slices, k = blockIdx.x / slices;
  const long long n = stat_images[k];
  const JitterDesc& d = descs[n];
  const Chain ch = load_chain(d, params + kParams * n);
  const Slice sl = pixel_slice(d, s, slices);
  const long long sc = d.sc;
  Acc acc = 0;
  for (long long p = sl.p0 + threadIdx.x; p < sl.p1; p += kThreads) {
    const T* px = pixel_at<T>(d, p);
    float r[1] = {(float)px[0]}, g[1] = {r[0]}, b[1] = {r[0]};
    if (ch.rgb) g[0] = (float)px[sc], b[0] = (float)px[2 * sc];
    run_ops<kU8, 1>(ch, 0, ch.at, 0.f, r, g, b);
    const float l = ch.rgb ? gray_px<kU8>(r[0], g[0], b[0]) : r[0];
    acc += kU8 ? (Acc)(int)l : (Acc)l;
  }
  const Acc sum = ordered_block_sum<kThreads>(acc);
  if (threadIdx.x == 0) static_cast<Acc*>(scratch)[(long long)k * slices + s] = sum;
}

__global__ void __launch_bounds__(kThreads) jitter_stats_kernel(const JitterDesc* __restrict__ descs,
                                                                const float* __restrict__ params,
                                                                const long long* __restrict__ stat_images,
                                                                void* scratch, int slices, int is_u8) {
  if (is_u8) stats_body<uint8_t>(descs, params, stat_images, scratch, slices);
  else stats_body<float>(descs, params, stat_images, scratch, slices);
}

template <typename T>
__device__ __forceinline__ void apply_body(const JitterDesc* __restrict__ descs, const float* __restrict__ params,
                                           const void* scratch, int slices, int rows_per_tile, int tiles) {
  constexpr bool kU8 = sizeof(T) == 1;
  constexpr int kVec = Vec16<T>::N;  // pixels per 16-byte vector: a chunk is kChunk / kVec vectors per channel
  const int n = blockIdx.x / tiles;
  const JitterDesc& d = descs[n];
  const Chain ch = load_chain(d, params + (long long)kParams * n);
  const int C = (int)d.C, H = (int)d.H, W = (int)d.W;
  float mean = 0.f;
  if (ch.at >= 0) {
    // the slice partials in slice order; torch's CUDA mean: the fp32 sum times its fp32 factor (outputs / inputs)
    if (kU8) {
      const long long* part = static_cast<const long long*>(scratch) + d.stat * slices;
      long long sum = 0;
      for (int s = 0; s < slices; ++s) sum += part[s];
      mean = (float)sum;
    } else {
      const double* part = static_cast<const double*>(scratch) + d.stat * slices;
      double sum = 0.0;
      for (int s = 0; s < slices; ++s) sum += part[s];
      mean = (float)sum;
    }
    mean = __fmul_rn(mean, ch.p[kMeanFactor]);
  }
  const T* src = reinterpret_cast<const T*>(d.src);
  T* dst = reinterpret_cast<T*>(d.dst);
  const long long sc = d.sc, sh = d.sh, sw = d.sw, plane = (long long)H * W;
  const RowTile tile(n, tiles, rows_per_tile, H, W);
  for (int item = threadIdx.x; item < tile.items(); item += kThreads) {
    const auto [y, x0, len] = Chunk(tile, item, W);
    const T* srow = src + y * sh + x0 * sw;
    T* drow = dst + ((long long)y * W + x0);
#pragma unroll 1
    for (int v0 = 0; v0 < len; v0 += kVec) {
      Vec16<T> v[3];
      const T* sp = srow + v0 * sw;
      v[0] = load_chunk(sp, sw, len - v0);
      v[1] = v[2] = v[0];
      if (C == 3) v[1] = load_chunk(sp + sc, sw, len - v0), v[2] = load_chunk(sp + 2 * sc, sw, len - v0);
      float r[kVec], g[kVec], b[kVec];
#pragma unroll
      for (int j = 0; j < kVec; ++j) r[j] = (float)v[0].v[j], g[j] = (float)v[1].v[j], b[j] = (float)v[2].v[j];
      run_ops<kU8, kVec>(ch, 0, ch.n, mean, r, g, b);
#pragma unroll
      for (int j = 0; j < kVec; ++j) v[0].v[j] = (T)r[j], v[1].v[j] = (T)g[j], v[2].v[j] = (T)b[j];
      store_chunk(drow + v0, v[0], len - v0);
      if (C == 3) store_chunk(drow + plane + v0, v[1], len - v0), store_chunk(drow + 2 * plane + v0, v[2], len - v0);
    }
  }
}

__global__ void __launch_bounds__(kThreads) jitter_apply_kernel(const JitterDesc* __restrict__ descs,
                                                                const float* __restrict__ params,
                                                                const void* scratch, int slices, int rows_per_tile,
                                                                int tiles, int is_u8) {
  if (is_u8) apply_body<uint8_t>(descs, params, scratch, slices, rows_per_tile, tiles);
  else apply_body<float>(descs, params, scratch, slices, rows_per_tile, tiles);
}

}  // namespace

extern "C" int hb_color_jitter_batch(const void* descs, const float* params, const long long* stat_images,
                                     void* scratch, int N, int n_stat, int H, int W, int slices, int dtype,
                                     void* stream) {
  if (N <= 0 || n_stat < 0 || n_stat > N || H <= 0 || W <= 0 || slices <= 0 ||
      (dtype != HB_DTYPE_F32 && dtype != HB_DTYPE_U8))
    return (int)cudaErrorInvalidValue;
  const auto* d = static_cast<const JitterDesc*>(descs);
  auto s = static_cast<cudaStream_t>(stream);
  const int is_u8 = dtype == HB_DTYPE_U8;
  if (n_stat > 0) {
    const long long blocks = (long long)n_stat * slices;
    if (blocks > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
    jitter_stats_kernel<<<(unsigned)blocks, kThreads, 0, s>>>(d, params, stat_images, scratch, slices, is_u8);
    HB_LAUNCH_CHECK();
  }
  int rows_per_tile, tiles;
  if (!row_tiles<kThreads>(N, H, W, rows_per_tile, tiles)) return (int)cudaErrorInvalidValue;
  jitter_apply_kernel<<<(unsigned)(N * tiles), kThreads, 0, s>>>(d, params, scratch, slices, rows_per_tile, tiles,
                                                                  is_u8);
  HB_LAUNCH_CHECK();
  return 0;
}
