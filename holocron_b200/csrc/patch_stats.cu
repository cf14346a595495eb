// Per-patch statistics for NormConv2d on the tensor cores (reference holocron/nn/functional.py:322-413: `unfold`, then each
// im2col patch - the whole Cin*kh*kw vector, zero padding included - is standardised with its biased variance).
// The reference materialises the N x L x (Cin*k*k) im2col tensor (9x the input) and makes two reduction passes over it.
// Here: one streaming pass reduces every input pixel over its channels (s1 = sum x, s2 = sum x^2), then every output pixel
// adds the kh*kw window entries of those two maps: mean = S1/K, var = S2/K - mean^2. The convolution itself runs on the
// implicit-GEMM tensor-core kernel (conv_fprop.cu) with the standardisation folded into its epilogue (hb_conv_args.norm_*).
#include <climits>

#include "common.cuh"

namespace {

using namespace hb;

// one thread per input pixel: C/8 128-bit vectors of bf16
__global__ void __launch_bounds__(256) pixel_moments_kernel(const __nv_bfloat16* __restrict__ x, float2* __restrict__ out,
                                                            long long npix, int C) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix) return;
  const __nv_bfloat16* p = x + i * C;
  float s1 = 0.f, s2 = 0.f;
  for (int c = 0; c < C; c += 8) {
    const Vec16<__nv_bfloat16> v = ld16(p + c);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float f = __bfloat162float(v.v[j]);
      s1 += f; s2 = fmaf(f, f, s2);
    }
  }
  out[i] = make_float2(s1, s2);
}

__global__ void __launch_bounds__(256) patch_stats_kernel(const float2* __restrict__ mom, float* __restrict__ mean,
                                                          float* __restrict__ rstd, int N, int H, int W, int Ho, int Wo, int kh,
                                                          int kw, int stride, int pad, int dil, float inv_k, float eps) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= (long long)N * Ho * Wo) return;
  const int wo = (int)(m % Wo), ho = (int)((m / Wo) % Ho), n = (int)(m / ((long long)Wo * Ho));
  double s1 = 0.0, s2 = 0.0;   // fp64 from here on: var = E[x^2] - mean^2 cancels when the patch mean dominates
  for (int r = 0; r < kh; ++r) {
    const int ih = ho * stride - pad + r * dil;
    if (ih < 0 || ih >= H) continue;
    for (int s = 0; s < kw; ++s) {
      const int iw = wo * stride - pad + s * dil;
      if (iw < 0 || iw >= W) continue;
      const float2 v = mom[((long long)n * H + ih) * W + iw];
      s1 += (double)v.x; s2 += (double)v.y;
    }
  }
  const double mu = s1 * (double)inv_k;
  double var = s2 * (double)inv_k - mu * mu;
  var = var < 0.0 ? 0.0 : var;
  mean[m] = (float)mu;
  rstd[m] = (float)(1.0 / sqrt(var + (double)eps));
}

}  // namespace

extern "C" int hb_patch_stats_bf16(const void* x, float* mean, float* rstd, float* scratch, int N, int H, int W, int C, int kh,
                                   int kw, int stride, int pad, int dil, int k_logical, float eps, void* stream) {
  if (C % 8 != 0 || !hb::aligned16(x) || !scratch) return (int)cudaErrorInvalidValue;
  // geometry, before any host division: positive sizes, a window window_out accepts on both axes, int-sized pixel and
  // patch counts, and a logical patch length (the unpadded Cin*kh*kw) no longer than the padded one
  int Ho, Wo;
  if (N <= 0 || C <= 0 || !hb::window_out(H, kh, stride, pad, dil, Ho) || !hb::window_out(W, kw, stride, pad, dil, Wo))
    return (int)cudaErrorInvalidValue;
  if ((long long)Ho * Wo > INT_MAX || (long long)N * Ho * Wo > INT_MAX) return (int)cudaErrorInvalidValue;
  if ((long long)C * kh > INT_MAX || (long long)C * kh * kw > INT_MAX || k_logical <= 0 || k_logical > C * kh * kw)
    return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  const long long npix = (long long)N * H * W, nout = (long long)N * Ho * Wo;
  pixel_moments_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, st>>>((const __nv_bfloat16*)x, (float2*)scratch, npix, C);
  HB_LAUNCH_CHECK();
  patch_stats_kernel<<<(unsigned)((nout + 255) / 256), 256, 0, st>>>((const float2*)scratch, mean, rstd, N, H, W, Ho, Wo, kh, kw,
                                                                    stride, pad, dil, 1.f / (float)k_logical, eps);
  HB_LAUNCH_CHECK();
  return 0;
}
