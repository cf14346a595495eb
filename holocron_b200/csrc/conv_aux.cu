// Small layout / helper kernels around the tensor-core convolutions (all HBM streaming passes):
//   * filter packing: fp32 KRSC master weights -> bf16 KRSC (channel padded) and the flipped+transposed
//     bf16 filter used by the data-gradient pass,
//   * zero insertion (stride-s transposed convolution input),
//   * NCHW fp32/bf16 image -> NHWC bf16 with channel padding (network input),
//   * global average pooling forward / backward over NHWC (reference holocron/nn/modules/downsample.py:58-74).
#include "common.cuh"

namespace {

using namespace hb;

// One filter to pack. w: [Cout][R][S][Cin] fp32.  wf: [CoutF][R][S][CinP] bf16 (zero padded).  wd (may be null):
// [CinD][R][S][CoutP] bf16 with wd[ci][r][s][co] = w[co][R-1-r][S-1-s][ci] (rows ci >= Cin and columns co >= Cout are zero).
struct PackMeta {
  const float* w;
  __nv_bfloat16* wf;
  __nv_bfloat16* wd;
  int Cout, Cin, R, S, CinP, CinD, CoutP, CoutF;

  __host__ __device__ size_t nf() const { return (size_t)CoutF * R * S * CinP; }
  __host__ __device__ size_t total() const { return nf() + (wd ? (size_t)CinD * R * S * CoutP : 0); }
};
constexpr int kPackChunk = 4096;

// Element i of the packed pair: wf[i] for i < nf, else wd[i - nf]. The divisions and the w offset run in the index type
// I (unsigned when the pair has fewer than 2^31 elements); the filter coordinates fit an int.
template <typename I>
__device__ __forceinline__ void pack_element(const PackMeta& m, I i, I nf) {
  const int R = m.R, S = m.S, Cin = m.Cin, Cout = m.Cout;
  if (i < nf) {
    const int ci = i % (I)m.CinP;
    I t = i / (I)m.CinP;
    const int s = t % S; t /= S;
    const int r = t % R;
    const int co = t / R;
    const float v = (ci < Cin && co < Cout) ? m.w[(((I)co * R + r) * S + s) * Cin + ci] : 0.f;
    m.wf[i] = __float2bfloat16_rn(v);
  } else {
    const I k = i - nf;
    const int co = k % (I)m.CoutP;
    I t = k / (I)m.CoutP;
    const int s = t % S; t /= S;
    const int r = t % R;
    const int ci = t / R;
    const float v = (co < Cout && ci < Cin) ? m.w[(((I)co * R + (R - 1 - r)) * S + (S - 1 - s)) * Cin + ci] : 0.f;
    m.wd[k] = __float2bfloat16_rn(v);
  }
}

__global__ void pack_weights_kernel(const __grid_constant__ PackMeta m) {
  const size_t nf = m.nf(), total = m.total();
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) pack_element<size_t>(m, i, nf);
}

// Multi-tensor variant: one launch packs every filter of a network (table row = one filter, chunk = 4096 output
// elements of one filter), instead of one launch per layer and step.
__global__ void __launch_bounds__(256) pack_weights_multi_kernel(const PackMeta* __restrict__ metas,
                                                                 const int2* __restrict__ chunks) {
  const int2 ck = chunks[blockIdx.x];
  const PackMeta m = metas[ck.x];
  const size_t nf = m.nf(), total = m.total();
  const size_t base = (size_t)ck.y * kPackChunk;
  const size_t end = min(base + (size_t)kPackChunk, total);
  if (total < 0x7fffffffu) {
    // every filter of a real network: 32-bit index arithmetic (the four runtime div/mod pairs per element dominated this kernel
    // when done on size_t: ALU bound, not memory bound, for RepVGG-A0's 18 M packed elements)
    for (unsigned i = (unsigned)base + threadIdx.x; i < (unsigned)end; i += 256) pack_element<unsigned>(m, i, (unsigned)nf);
    return;
  }
  for (size_t i = base + threadIdx.x; i < end; i += 256) pack_element<size_t>(m, i, nf);
}

// Class filters of the stride-2 3x3 pad-1 data gradient (hb_conv2d_dgrad_s2_bf16). Output parity class (a, b) is a
// correlation over dy with (1+a) x (1+b) taps: out_ab[ci][t][u][co] = w[co][r(a,t)][s(b,u)][ci] with
// r(0,0) = 1, r(1,0) = 2, r(1,1) = 0 (dy row i+t feeds dx row 2i+a through filter row r = 2i+a+1-2(i+t)).
// Classes are stored back to back in the order (0,0), (0,1), (1,0), (1,1); rows ci >= Cin / columns co >= Cout are zero.
__global__ void pack_dgrad_s2_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ out, int Cout, int Cin,
                                     int CinD, int CoutP) {
  const size_t unit = (size_t)CinD * CoutP;
  const size_t total = 9 * unit;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    int a, b; size_t k;
    if (i < unit) { a = 0; b = 0; k = i; }
    else if (i < 3 * unit) { a = 0; b = 1; k = i - unit; }
    else if (i < 5 * unit) { a = 1; b = 0; k = i - 3 * unit; }
    else { a = 1; b = 1; k = i - 5 * unit; }
    const int S = 1 + b, R = 1 + a;
    const int co = k % CoutP;
    size_t t = k / CoutP;
    const int u = t % S; t /= S;
    const int tt = t % R;
    const int ci = t / R;
    const int r = a == 0 ? 1 : (tt == 0 ? 2 : 0);
    const int sx = b == 0 ? 1 : (u == 0 ? 2 : 0);
    const float v = (co < Cout && ci < Cin) ? w[(((size_t)co * 3 + r) * 3 + sx) * Cin + ci] : 0.f;
    out[i] = __float2bfloat16_rn(v);
  }
}

// y[n, sp*p, sp*q, :] = x[n, p, q, :]; everything else zero. One thread per 16-byte channel vector of y.
__global__ void zero_insert_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int N, int Hi,
                                   int Wi, int Ho, int Wo, int C, int sp) {
  const int cv = C / 8;
  const size_t total = (size_t)N * Ho * Wo * cv;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int c = i % cv;
    size_t t = i / cv;
    const int w = t % Wo; t /= Wo;
    const int h = t % Ho;
    const int n = t / Ho;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (h % sp == 0 && w % sp == 0) {
      const int p = h / sp, q = w / sp;
      if (p < Hi && q < Wi) v = *reinterpret_cast<const uint4*>(x + (((size_t)n * Hi + p) * Wi + q) * C + c * 8);
    }
    *reinterpret_cast<uint4*>(y + i * 8) = v;
  }
}

template <typename T>
__global__ void nchw_to_nhwc_pad_kernel(const T* __restrict__ x, __nv_bfloat16* __restrict__ y, int N, int C, int HW,
                                        int CP) {
  // one thread per output pixel: reads C strided planes (coalesced across threads), writes CP contiguous bf16
  const size_t total = (size_t)N * HW;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const size_t n = i / HW, p = i % HW;
    for (int c0 = 0; c0 < CP; c0 += 8) {
      Vec16<__nv_bfloat16> o;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = c0 + j;
        o.v[j] = c < C ? from_f<__nv_bfloat16>(to_f(x[(n * C + c) * HW + p])) : __float2bfloat16_rn(0.f);
      }
      st16(y + i * CP + c0, o);
    }
  }
}

// Explicit im2col for convolutions with a handful of input channels (network stems, Cin <= 4): the implicit-GEMM
// kernels would pad such a Cin to a 64-channel K block (>= 87% of the tensor-core and TMA work wasted on
// RepVGG's 3->48 stem). Here the R*S*C patch of every output pixel is written once as one dense row of
// Kp = 32 (or 64) bf16 values, k = (r*S + s)*C + c, and the convolution becomes a plain [M, Kp] x [Kp, Cout] GEMM on the
// tensor-core kernel (forward) / its wgrad twin (backward). x: NCHW of any float dtype.
template <typename T>
__global__ void im2col_smallc_kernel(const T* __restrict__ x, __nv_bfloat16* __restrict__ col, int N, int C, int H, int W,
                                     int Ho, int Wo, int R, int S, int stride, int pad, int Kp) {
  const size_t total = (size_t)N * Ho * Wo;
  const size_t tstride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += tstride) {
    const int wo = (int)(i % Wo);
    const int ho = (int)((i / Wo) % Ho);
    const size_t n = i / ((size_t)Wo * Ho);
    __nv_bfloat16* dst = col + i * Kp;
    for (int k0 = 0; k0 < Kp; k0 += 8) {
      Vec16<__nv_bfloat16> o;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int k = k0 + j;
        float v = 0.f;
        if (k < R * S * C) {
          const int c = k % C, tap = k / C;
          const int r = tap / S, s = tap % S;
          const int hi = ho * stride + r - pad, wi = wo * stride + s - pad;
          if (hi >= 0 && hi < H && wi >= 0 && wi < W) v = to_f(x[((n * C + c) * H + hi) * W + wi]);
        }
        o.v[j] = __float2bfloat16_rn(v);
      }
      st16(dst + k0, o);
    }
  }
}

// The usual stem (3 channels, 3x3, Kp = 32) with everything known at compile time: no integer divisions per element.
template <typename T>
__global__ void im2col_c3k3_kernel(const T* __restrict__ x, __nv_bfloat16* __restrict__ col, int N, int H, int W, int Ho,
                                   int Wo, int stride, int pad) {
  const size_t total = (size_t)N * Ho * Wo;
  const size_t tstride = (size_t)gridDim.x * blockDim.x;
  const size_t plane = (size_t)H * W;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += tstride) {
    const unsigned iu = (unsigned)i;              // total < 2^32 checked by the launcher: 32-bit divisions
    const unsigned t1 = iu / (unsigned)Wo;
    const int wo = (int)(iu - t1 * (unsigned)Wo);
    const size_t n = t1 / (unsigned)Ho;
    const int ho = (int)(t1 - (unsigned)n * (unsigned)Ho);
    const T* xn = x + n * 3 * plane;
    float v[32];
#pragma unroll
    for (int k = 27; k < 32; ++k) v[k] = 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int hi = ho * stride + r - pad;
      const bool hok = hi >= 0 && hi < H;
#pragma unroll
      for (int s2 = 0; s2 < 3; ++s2) {
        const int wi = wo * stride + s2 - pad;
        const bool ok = hok && wi >= 0 && wi < W;
        const size_t o = (size_t)hi * W + wi;
#pragma unroll
        for (int c = 0; c < 3; ++c) v[(r * 3 + s2) * 3 + c] = ok ? to_f(xn[c * plane + o]) : 0.f;
      }
    }
    __nv_bfloat16* dst = col + i * 32;
#pragma unroll
    for (int k0 = 0; k0 < 32; k0 += 8) {
      Vec16<__nv_bfloat16> o;
#pragma unroll
      for (int j = 0; j < 8; ++j) o.v[j] = __float2bfloat16_rn(v[k0 + j]);
      st16(dst + k0, o);
    }
  }
}

// GAP backward: dx[n, r, c] = dy[n, c] / HW
__global__ void gap_bwd_kernel(const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ dx, int N, int HW, int C) {
  const int cv = C / 8;
  const size_t total = (size_t)N * HW * cv;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const float inv = 1.f / (float)HW;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const size_t c = i % cv;
    const size_t n = i / ((size_t)HW * cv);
    Vec16<__nv_bfloat16> v = ld16(dy + n * C + c * 8), o;
#pragma unroll
    for (int j = 0; j < 8; ++j) o.v[j] = __float2bfloat16_rn(__bfloat162float(v.v[j]) * inv);
    st16(dx + i * 8, o);
  }
}

}  // namespace

extern "C" {

int hb_pack_conv_weights(const float* w, void* wf, void* wd, int Cout, int Cin, int R, int S, int CinP, int CinD,
                         int CoutP, int CoutF, void* stream) {
  if (CoutF < Cout || CinP < Cin) return (int)cudaErrorInvalidValue;
  const PackMeta m{w, (__nv_bfloat16*)wf, (__nv_bfloat16*)wd, Cout, Cin, R, S, CinP, CinD, CoutP, CoutF};
  const size_t n = m.total();
  if (n == 0) return 0;
  pack_weights_kernel<<<stream_grid(n, 256), 256, 0, (cudaStream_t)stream>>>(m);
  HB_LAUNCH_CHECK();
  return 0;
}

// metas: device array of 64-byte rows {w, wf, wd, Cout, Cin, R, S, CinP, CinD, CoutP, CoutF} (3 pointers + 8 int32, padded
// to 64 bytes); chunks: device array of int32 pairs (row, chunk index) with hb_pack_chunk_elems() elements per chunk.
int hb_pack_conv_weights_multi(const void* metas, const void* chunks, int num_chunks, void* stream) {
  static_assert(sizeof(PackMeta) == 56 || sizeof(PackMeta) == 64, "PackMeta layout");
  if (num_chunks <= 0) return 0;
  pack_weights_multi_kernel<<<num_chunks, 256, 0, (cudaStream_t)stream>>>((const PackMeta*)metas, (const int2*)chunks);
  HB_LAUNCH_CHECK();
  return 0;
}
int hb_pack_chunk_elems(void) { return kPackChunk; }
int hb_pack_meta_bytes(void) { return (int)sizeof(PackMeta); }

int hb_pack_dgrad_s2_weights(const float* w, void* out, int Cout, int Cin, int CinD, int CoutP, void* stream) {
  if (CinD < Cin || CoutP < Cout) return (int)cudaErrorInvalidValue;
  const size_t n = (size_t)9 * CinD * CoutP;
  if (n == 0) return 0;
  pack_dgrad_s2_kernel<<<stream_grid(n, 256), 256, 0, (cudaStream_t)stream>>>(w, (__nv_bfloat16*)out, Cout, Cin, CinD, CoutP);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_zero_insert_bf16(const void* x, void* y, int N, int Hi, int Wi, int Ho, int Wo, int C, int sp, void* stream) {
  if (C % 8 != 0) return (int)cudaErrorInvalidValue;
  const size_t n = (size_t)N * Ho * Wo * (C / 8);
  if (n == 0) return 0;
  zero_insert_kernel<<<stream_grid(n, 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y,
                                                                            N, Hi, Wi, Ho, Wo, C, sp);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_nchw_to_nhwc_pad_bf16(const void* x, void* y, int N, int C, int H, int W, int CP, int dtype, void* stream) {
  if (CP % 8 != 0 || CP < C) return (int)cudaErrorInvalidValue;
  const size_t n = (size_t)N * H * W;
  if (n == 0) return 0;
  const int grid = stream_grid(n, 256);
  return dispatch_dtype(dtype, [&](auto type) {
    using T = typename decltype(type)::type;
    nchw_to_nhwc_pad_kernel<T><<<grid, 256, 0, (cudaStream_t)stream>>>((const T*)x, (__nv_bfloat16*)y, N, C, H * W, CP);
    HB_LAUNCH_CHECK();
    return 0;
  });
}

int hb_im2col_smallc_bf16(const void* x, void* col, int N, int C, int H, int W, int R, int S, int stride, int pad, int Kp,
                          int dtype, void* stream) {
  if (Kp % 8 != 0 || Kp < R * S * C) return (int)cudaErrorInvalidValue;
  int Ho, Wo;
  if (!window_out(H, R, stride, pad, 1, Ho) || !window_out(W, S, stride, pad, 1, Wo)) return (int)cudaErrorInvalidValue;
  const size_t n = (size_t)N * Ho * Wo;
  if (n == 0) return 0;
  const int grid = stream_grid(n, 256, 16);
  cudaStream_t st = (cudaStream_t)stream;
  __nv_bfloat16* c = (__nv_bfloat16*)col;
  return dispatch_dtype(dtype, [&](auto type) {
    using T = typename decltype(type)::type;
    if (C == 3 && R == 3 && S == 3 && Kp == 32 && n < 0xffffffffull)
      im2col_c3k3_kernel<T><<<grid, 256, 0, st>>>((const T*)x, c, N, H, W, Ho, Wo, stride, pad);
    else
      im2col_smallc_kernel<T><<<grid, 256, 0, st>>>((const T*)x, c, N, C, H, W, Ho, Wo, R, S, stride, pad, Kp);
    HB_LAUNCH_CHECK();
    return 0;
  });
}

int hb_gap_bwd_bf16(const void* dy, void* dx, int N, int HW, int C, void* stream) {
  if (C % 8 != 0) return (int)cudaErrorInvalidValue;
  const size_t n = (size_t)N * HW * (C / 8);
  if (n == 0) return 0;
  gap_bwd_kernel<<<stream_grid(n, 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)dy, (__nv_bfloat16*)dx, N,
                                                                        HW, C);
  HB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
