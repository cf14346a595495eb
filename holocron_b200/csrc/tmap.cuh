// Host-side CUtensorMap construction. The driver entry points are resolved at run time with
// cudaGetDriverEntryPoint so the library has no link-time dependency on libcuda.
#pragma once
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

namespace tmap {

struct Api {
  PFN_cuTensorMapEncodeTiled_v12000 tiled = nullptr;
  PFN_cuTensorMapEncodeIm2col_v12000 im2col = nullptr;
  int driver_version = 0;
  bool ok = false;
};

inline const Api& api() {
  static Api a = [] {
    Api r;
    cudaDriverEntryPointQueryResult q;
    void* f = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      r.tiled = (PFN_cuTensorMapEncodeTiled_v12000)f;
    f = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &f, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      r.im2col = (PFN_cuTensorMapEncodeIm2col_v12000)f;
    cudaDriverGetVersion(&r.driver_version);
    r.ok = r.tiled && r.im2col;
    return r;
  }();
  return a;
}

// Row-major bf16 tensor of `rank` dims; dims[0] is the contiguous one. strides_bytes[i] is the byte stride
// of dim i+1 (rank-1 entries). box[i] <= 256, box[0]*2 bytes <= swizzle span.
inline int encode_tiled_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                             const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swz) {
  const Api& a = api();
  if (!a.ok) return (int)cudaErrorNotSupported;
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = a.tiled(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base),
                       (const cuuint64_t*)dims, (const cuuint64_t*)strides_bytes, (const cuuint32_t*)box, estr,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)cudaErrorInvalidValue;
}

// The tiled maps of the tensor-core convolutions. Every box is 64 channels wide (one 128-byte swizzle row).
// NHWC tensor [N, H, W, C]: box of box_w pixels x box_h rows of one image.
inline int encode_nhwc_box(CUtensorMap* out, const void* base, int N, int H, int W, int C, uint32_t box_w,
                           uint32_t box_h) {
  const uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)N};
  const uint64_t strides[3] = {(uint64_t)C * 2, (uint64_t)W * C * 2, (uint64_t)H * W * C * 2};
  const uint32_t box[4] = {64, box_w, box_h, 1};
  return encode_tiled_bf16(out, base, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}
// KRSC filter [K, taps, C]: the slab of one tap for box_k filters.
inline int encode_krsc_slab(CUtensorMap* out, const void* base, int K, int taps, int C, uint32_t box_k) {
  const uint64_t dims[3] = {(uint64_t)C, (uint64_t)taps, (uint64_t)K};
  const uint64_t strides[2] = {(uint64_t)C * 2, (uint64_t)taps * C * 2};
  const uint32_t box[3] = {64, 1, box_k};
  return encode_tiled_bf16(out, base, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}
// Row-major matrix [M, C]: box of box_m rows.
inline int encode_matrix(CUtensorMap* out, const void* base, int M, int C, uint32_t box_m) {
  const uint64_t dims[2] = {(uint64_t)C, (uint64_t)M};
  const uint64_t strides[1] = {(uint64_t)C * 2};
  const uint32_t box[2] = {64, box_m};
  return encode_tiled_bf16(out, base, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

// im2col map over an NHWC bf16 activation tensor (TMA dims C, W, H, N).
//   lower corner = -pad, upper corner = pad - (k-1)*dil  (the box the filter's top-left tap may visit);
//   traversal stride = conv stride. channels/pixels per load = the smem tile (64 x 128 here).
inline int encode_im2col_bf16(CUtensorMap* out, const void* base, int N, int H, int W, int C, int pad_h, int pad_w,
                              int kh, int kw, int dil, int stride, uint32_t channels_per_pixel,
                              uint32_t pixels_per_column, CUtensorMapSwizzle swz, int pad_after_h = -1,
                              int pad_after_w = -1) {
  const Api& a = api();
  if (pad_after_h < 0) pad_after_h = pad_h;   // symmetric padding unless stated
  if (pad_after_w < 0) pad_after_w = pad_w;
  if (!a.ok) return (int)cudaErrorNotSupported;
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  int lower[2] = {-pad_w, -pad_h};
  int upper[2] = {pad_after_w - (kw - 1) * dil, pad_after_h - (kh - 1) * dil};
  cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  CUresult r = a.im2col(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, lower, upper,
                        channels_per_pixel, pixels_per_column, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return (int)cudaErrorInvalidValue;
  // Known driver issue (also worked around by CUTLASS' im2col descriptor builder): for tensors smaller
  // than 128 KiB, drivers <= 13.1 set a descriptor bit that makes im2col loads fault.
  if (a.driver_version <= 13010 && (uint64_t)N * H * W * C * 2 < 131072ull) {
    reinterpret_cast<uint64_t*>(out)[1] &= ~(1ull << 21);
  }
  return 0;
}

}  // namespace tmap
