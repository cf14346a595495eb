// DropBlock (reference holocron/nn/functional.py:465-500, nn/modules/dropblock.py:14-41).
//   mask[n,h,w] = 1 - max_{bs x bs window, stride 1, pad bs/2}(noise <= gamma)   (shared across channels)
//   out = x * mask * (mask.numel() / mask.sum())            (rescale skipped when mask.sum() == 0)
// The reference needs rand + max_pool2d + 2 multiplies + a host sync on mask.sum(); here: one mask/count kernel
// (N*H*W sized) and one apply pass over x, the rescale factor staying on the device.
// The kept count is an integer (exact and independent of block order at any size); the scale is rounded as the
// reference's `int / Tensor` rounds it: torch evaluates numel / kept as kept.reciprocal() * numel, two fp32 roundings.
#include "common.cuh"

namespace {

using namespace hb;

__global__ void dropblock_mask_kernel(const float* __restrict__ noise, float* __restrict__ mask,
                                      unsigned long long* __restrict__ kept, int N, int H, int W, int bs, float gamma) {
  const long long total = (long long)N * H * W;
  const int half = bs / 2;
  // a thread counts at most ceil(total / (grid * 256)) cells and a warp 32 times that: far below 2^32 for any mask
  // that fits in device memory
  unsigned local = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int w = (int)(i % W);
    const int h = (int)((i / W) % H);
    const long long n = i / ((long long)W * H);
    bool hit = false;
    for (int dh = -half; dh <= half && !hit; ++dh) {
      const int hh = h + dh;
      if (hh < 0 || hh >= H) continue;
      for (int dw = -half; dw <= half; ++dw) {
        const int ww = w + dw;
        if (ww < 0 || ww >= W) continue;
        if (noise[(n * H + hh) * W + ww] <= gamma) { hit = true; break; }
      }
    }
    mask[i] = hit ? 0.f : 1.f;
    local += hit ? 0u : 1u;
  }
  const unsigned warp = __reduce_add_sync(0xffffffffu, local);
  if ((threadIdx.x & 31) == 0 && warp != 0) atomicAdd(kept, (unsigned long long)warp);
}

// numel / kept as the reference rounds it (fl(fl(1 / kept) * numel)), 1 when nothing is kept
__device__ __forceinline__ float dropblock_scale(const unsigned long long* kept, float numel) {
  const float k = __ull2float_rn(*kept);
  return k > 0.f ? __fmul_rn(__frcp_rn(k), numel) : 1.f;
}

// x is [N, C, H, W] logical; channels_last != 0 -> physical NHWC. out may alias x.
template <typename T>
__global__ void dropblock_apply_kernel(const T* x, T* out, const float* __restrict__ mask,
                                       const unsigned long long* __restrict__ kept, long long total, int C, long long HW,
                                       int channels_last, float numel) {
  const float scale = dropblock_scale(kept, numel);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long mi;
    if (channels_last) {
      mi = i / C;                       // (n*HW + hw)
    } else {
      const long long n = i / ((long long)C * HW);
      mi = n * HW + (i % HW);
    }
    out[i] = from_f<T>(to_f(x[i]) * mask[mi] * scale);
  }
}

// channels_last fast path: one 128-bit vector (16 / sizeof(T) channels of one pixel) per thread step, 32-bit index arithmetic
// (the scalar kernel above does a 64-bit division per ELEMENT; YOLOv4 has a DropBlock behind every conv)
template <typename T>
__global__ void __launch_bounds__(256) dropblock_apply_nhwc_vec_kernel(const T* x, T* out, const float* __restrict__ mask,
                                                                       const unsigned long long* __restrict__ kept,
                                                                       unsigned total_vec, unsigned cvec, float numel) {
  const float scale = dropblock_scale(kept, numel);
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total_vec; i += gridDim.x * blockDim.x) {
    const float m = __ldg(mask + i / cvec) * scale;
    Vec16<T> v = ld16(x + (size_t)i * Vec16<T>::N);
#pragma unroll
    for (int j = 0; j < Vec16<T>::N; ++j) v.v[j] = from_f<T>(to_f(v.v[j]) * m);
    st16(out + (size_t)i * Vec16<T>::N, v);
  }
}

template <typename T>
bool launch_nhwc_vec(const void* x, void* out, const float* mask, const unsigned long long* kept, long long total, int C,
                     float numel, cudaStream_t st) {
  constexpr int V = Vec16<T>::N;
  if (C % V != 0 || !aligned16(x) || !aligned16(out) || total / V >= 0xffffffffLL) return false;
  const unsigned total_vec = (unsigned)(total / V);
  dropblock_apply_nhwc_vec_kernel<T><<<stream_grid((size_t)total_vec, 256 * 2), 256, 0, st>>>(
      (const T*)x, (T*)out, mask, kept, total_vec, (unsigned)(C / V), numel);
  return true;
}

}  // namespace

extern "C" {

// kept: device 64-bit count of the kept cells, zeroed here. mask: float[N*H*W]. block_size must be odd (as in the
// reference, where an even size makes the pooled mask one pixel larger than the input and the multiply fail).
int hb_dropblock_mask(const float* noise, float* mask, unsigned long long* kept, int N, int H, int W, int block_size,
                      float gamma, void* stream) {
  if (block_size % 2 == 0) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(kept, 0, sizeof(unsigned long long), st);
  if (e != cudaSuccess) return (int)e;
  const long long total = (long long)N * H * W;
  if (total == 0) return 0;
  dropblock_mask_kernel<<<stream_grid((size_t)total, 256), 256, 0, st>>>(noise, mask, kept, N, H, W, block_size, gamma);
  HB_LAUNCH_CHECK();
  return 0;
}

// out = x * mask * numel(mask)/kept; also the backward (x := upstream gradient).
int hb_dropblock_apply(const void* x, void* out, const float* mask, const unsigned long long* kept, int N, int C, int H,
                       int W, int channels_last, int dtype, void* stream) {
  const long long total = (long long)N * C * H * W;
  if (total == 0) return 0;
  const long long HW = (long long)H * W;
  const float numel = (float)((long long)N * HW);
  const int grid = stream_grid((size_t)total, 256 * 4);
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_dtype(dtype, [&](auto type) {
    using T = typename decltype(type)::type;
    if (!(channels_last && launch_nhwc_vec<T>(x, out, mask, kept, total, C, numel, st)))
      dropblock_apply_kernel<T><<<grid, 256, 0, st>>>((const T*)x, (T*)out, mask, kept, total, C, HW, channels_last, numel);
    HB_LAUNCH_CHECK();
    return 0;
  });
}

}  // extern "C"
