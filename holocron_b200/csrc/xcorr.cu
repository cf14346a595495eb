// Patch-wise cross-correlation family: NormConv2d and Add2d (AdderNet).
// Reference: holocron/nn/functional.py:322-462 (_xcorr2d / _convNd / norm_conv2d / _addNd / add2d).
//
//   patches p[n, l, k] = im2col(x) with k = (c, r, s) channel-major (the order of F.unfold), zero padding included;
//   optional slice normalisation: p <- (p - mean_k p) * rsqrt(var_k p + eps)   (biased variance over the WHOLE
//   Cin*kh*kw vector, zero padding participating - reference functional.py:346-349);
//   norm_conv2d: out[n, co, l] = sum_k p * w[co, k] (+ bias)
//   add2d      : out[n, co, l] = - sum_k |p - w[co, k]| (+ bias)          (no multiplies: CUDA cores, not tensor cores)
//
// The reference materialises the 9x-sized im2col tensor (and for add2d an N x L x Cout x K broadcast tensor). Here
// nothing is materialised: patches are gathered straight from x into shared-memory tiles (fp32, exact arithmetic
// so results match the fp32 reference to rounding), 32 x 32 output tiles per CTA, 2 x 2 outputs per thread.
// `groups` is ignored exactly as the reference ignores it.
#include <climits>

#include "common.cuh"

namespace {

constexpr int TL = 32;   // patches per tile
constexpr int TC = 32;   // output channels per tile
constexpr int TK = 32;   // reduction chunk

struct XcParams {
  int N, Cin, H, W, Cout, KH, KW, Ho, Wo, stride, pad, dil;
  int K;       // Cin*KH*KW
  int L;       // Ho*Wo
  int normalize;
  float eps;
};

__device__ __forceinline__ float patch_elem(const float* __restrict__ x, const XcParams& p, int n, int l, int k) {
  const int s = k % p.KW;
  const int r = (k / p.KW) % p.KH;
  const int c = k / (p.KW * p.KH);
  const int ho = l / p.Wo, wo = l % p.Wo;
  const int h = ho * p.stride - p.pad + r * p.dil;
  const int w = wo * p.stride - p.pad + s * p.dil;
  if (h < 0 || h >= p.H || w < 0 || w >= p.W) return 0.f;
  return x[(((size_t)n * p.Cin + c) * p.H + h) * p.W + w];
}

// per-patch mean and rsqrt(var + eps): one warp per patch
__global__ void patch_stats_kernel(const float* __restrict__ x, XcParams p, float* __restrict__ mean, float* __restrict__ rstd) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long total = (long long)p.N * p.L;
  if (warp >= total) return;
  const int n = (int)(warp / p.L), l = (int)(warp % p.L);
  float s = 0.f;
  for (int k = lane; k < p.K; k += 32) s += patch_elem(x, p, n, l, k);
  s = hb::warp_sum(s);
  const float mu = s / (float)p.K;
  float q = 0.f;
  for (int k = lane; k < p.K; k += 32) { const float d = patch_elem(x, p, n, l, k) - mu; q += d * d; }
  q = hb::warp_sum(q);
  if (lane == 0) { mean[warp] = mu; rstd[warp] = 1.0f / sqrtf(q / (float)p.K + p.eps); }
}

template <bool kAdder>
__global__ void __launch_bounds__(256) xcorr_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                        const float* __restrict__ bias, const float* __restrict__ mean,
                                                        const float* __restrict__ rstd, float* __restrict__ out, XcParams p) {
  __shared__ float sp[TK][TL + 1];  // [k][l]
  __shared__ float sw[TK][TC + 1];  // [k][co]
  const int n = blockIdx.z;
  const int l0 = blockIdx.x * TL, c0 = blockIdx.y * TC;
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;  // tx -> l pair, ty -> co pair
  float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  for (int k0 = 0; k0 < p.K; k0 += TK) {
    for (int i = threadIdx.x; i < TK * TL; i += 256) {
      const int kk = i / TL, ll = i % TL;
      const int k = k0 + kk, l = l0 + ll;
      float v = 0.f;
      if (k < p.K && l < p.L) {
        v = patch_elem(x, p, n, l, k);
        if (p.normalize) v = (v - mean[(size_t)n * p.L + l]) * rstd[(size_t)n * p.L + l];
      }
      sp[kk][ll] = v;
    }
    for (int i = threadIdx.x; i < TK * TC; i += 256) {
      const int cc = i / TK, kk = i % TK;
      const int k = k0 + kk, co = c0 + cc;
      sw[kk][cc] = (k < p.K && co < p.Cout) ? w[(size_t)co * p.K + k] : 0.f;
    }
    __syncthreads();
    const int kmax = min(TK, p.K - k0);
    for (int kk = 0; kk < kmax; ++kk) {
      const float a0 = sp[kk][tx * 2], a1 = sp[kk][tx * 2 + 1];
      const float b0 = sw[kk][ty * 2], b1 = sw[kk][ty * 2 + 1];
      if (kAdder) {
        acc[0][0] -= fabsf(a0 - b0); acc[0][1] -= fabsf(a0 - b1);
        acc[1][0] -= fabsf(a1 - b0); acc[1][1] -= fabsf(a1 - b1);
      } else {
        acc[0][0] = fmaf(a0, b0, acc[0][0]); acc[0][1] = fmaf(a0, b1, acc[0][1]);
        acc[1][0] = fmaf(a1, b0, acc[1][0]); acc[1][1] = fmaf(a1, b1, acc[1][1]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int l = l0 + tx * 2 + i, co = c0 + ty * 2 + j;
      if (l < p.L && co < p.Cout) out[((size_t)n * p.Cout + co) * p.L + l] = acc[i][j] + (bias ? bias[co] : 0.f);
    }
}

// dW[co, k] = sum_{n,l} g[n,co,l] * h(p[n,l,k], w[co,k]);  h = p (norm_conv) or sign(p - w) (adder: d(-|p-w|)/dw)
// grid: (k tiles, co tiles, splits over n*l); atomicAdd into zeroed dW
template <bool kAdder>
__global__ void __launch_bounds__(256) xcorr_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                          const float* __restrict__ g, const float* __restrict__ mean,
                                                          const float* __restrict__ rstd, float* __restrict__ dw, XcParams p,
                                                          int chunks_per_split) {
  __shared__ float sp[TL][TK + 1];  // [m][k]
  __shared__ float sg[TL][TC + 1];  // [m][co]
  const int k0 = blockIdx.x * TK, c0 = blockIdx.y * TC;
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;  // tx -> k pair, ty -> co pair
  const long long M = (long long)p.N * p.L;
  float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  float wv[2][2];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int k = k0 + tx * 2 + i, co = c0 + ty * 2 + j;
      wv[i][j] = (k < p.K && co < p.Cout) ? w[(size_t)co * p.K + k] : 0.f;
    }
  const long long m_begin = (long long)blockIdx.z * chunks_per_split * TL;
  const long long m_end = min(M, m_begin + (long long)chunks_per_split * TL);
  for (long long m0 = m_begin; m0 < m_end; m0 += TL) {
    for (int i = threadIdx.x; i < TL * TK; i += 256) {
      const int mm = i / TK, kk = i % TK;
      const long long m = m0 + mm;
      const int k = k0 + kk;
      float v = 0.f;
      if (m < m_end && k < p.K) {
        const int n = (int)(m / p.L), l = (int)(m % p.L);
        v = patch_elem(x, p, n, l, k);
        if (p.normalize) v = (v - mean[m]) * rstd[m];
      }
      sp[mm][kk] = v;
    }
    for (int i = threadIdx.x; i < TL * TC; i += 256) {
      const int cc = i / TL, mm = i % TL;
      const long long m = m0 + mm;
      const int co = c0 + cc;
      float v = 0.f;
      if (m < m_end && co < p.Cout) {
        const int n = (int)(m / p.L), l = (int)(m % p.L);
        v = g[((size_t)n * p.Cout + co) * p.L + l];
      }
      sg[mm][cc] = v;
    }
    __syncthreads();
    const int mmax = (int)min((long long)TL, m_end - m0);
    for (int mm = 0; mm < mmax; ++mm) {
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float pv = sp[mm][tx * 2 + i], gv = sg[mm][ty * 2 + j];
          if (kAdder) {
            const float d = pv - wv[i][j];
            acc[i][j] += gv * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
          } else {
            acc[i][j] = fmaf(gv, pv, acc[i][j]);
          }
        }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int k = k0 + tx * 2 + i, co = c0 + ty * 2 + j;
      if (k < p.K && co < p.Cout) atomicAdd(&dw[(size_t)co * p.K + k], acc[i][j]);
    }
}

// add2d (no slice normalisation): dx[n,c,h,w] = - sum_{r,s valid} sum_co g[n,co,ho,wo] * sign(x[n,c,h,w] - w[co,c,r,s])
__global__ void adder_dgrad_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ g,
                                   float* __restrict__ dx, XcParams p) {
  const long long total = (long long)p.N * p.Cin * p.H * p.W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int wi = (int)(i % p.W);
    const int hi = (int)((i / p.W) % p.H);
    const int c = (int)((i / ((long long)p.W * p.H)) % p.Cin);
    const int n = (int)(i / ((long long)p.W * p.H * p.Cin));
    const float xv = x[i];
    float acc = 0.f;
    for (int r = 0; r < p.KH; ++r) {
      const int hn = hi + p.pad - r * p.dil;
      if (hn < 0 || hn % p.stride != 0) continue;
      const int ho = hn / p.stride;
      if (ho >= p.Ho) continue;
      for (int s = 0; s < p.KW; ++s) {
        const int wn = wi + p.pad - s * p.dil;
        if (wn < 0 || wn % p.stride != 0) continue;
        const int wo = wn / p.stride;
        if (wo >= p.Wo) continue;
        const int k = (c * p.KH + r) * p.KW + s;
        for (int co = 0; co < p.Cout; ++co) {
          const float d = xv - w[(size_t)co * p.K + k];
          const float sg = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
          acc -= g[(((size_t)n * p.Cout + co) * p.Ho + ho) * p.Wo + wo] * sg;
        }
      }
    }
    dx[i] = acc;
  }
}

// Fills p when the geometry is accepted, checked before any host division or device call: positive sizes, a window
// window_out accepts on both axes, and int-sized pixel (N*Ho*Wo) and patch (Cin*KH*KW) counts.
bool make_params(XcParams& p, int N, int Cin, int H, int W, int Cout, int KH, int KW, int stride, int pad, int dil,
                 int normalize, float eps) {
  if (N <= 0 || Cin <= 0 || Cout <= 0) return false;
  int Ho, Wo;
  if (!hb::window_out(H, KH, stride, pad, dil, Ho) || !hb::window_out(W, KW, stride, pad, dil, Wo)) return false;
  if ((long long)Ho * Wo > INT_MAX || (long long)N * Ho * Wo > INT_MAX) return false;
  if ((long long)Cin * KH > INT_MAX || (long long)Cin * KH * KW > INT_MAX) return false;
  p = XcParams{N, Cin, H, W, Cout, KH, KW, Ho, Wo, stride, pad, dil, Cin * KH * KW, Ho * Wo, normalize, eps};
  return true;
}

}  // namespace

extern "C" {

// x fp32 NCHW, w fp32 [Cout,Cin,KH,KW], out fp32 [N,Cout,Ho,Wo]; mode 0: norm_conv (multiply-accumulate), 1: adder.
// mean/rstd: fp32 [N*Ho*Wo] scratch, written when normalize != 0 (kept for the backward).
int hb_xcorr2d_fwd(const float* x, const float* w, const float* bias, float* out, float* mean, float* rstd, int N, int Cin,
                   int H, int W, int Cout, int KH, int KW, int stride, int pad, int dil, int mode, int normalize,
                   float eps, void* stream) {
  // grid: (L tiles, Cout tiles, N)
  XcParams p;
  if (!make_params(p, N, Cin, H, W, Cout, KH, KW, stride, pad, dil, normalize, eps) || N > 65535 ||
      (Cout + TC - 1) / TC > 65535)
    return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  if (normalize) {
    const long long warps = (long long)N * p.L;
    patch_stats_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(x, p, mean, rstd);
    HB_LAUNCH_CHECK();
  }
  dim3 grid((p.L + TL - 1) / TL, (Cout + TC - 1) / TC, N);
  if (mode == 1) xcorr_fwd_kernel<true><<<grid, 256, 0, st>>>(x, w, bias, mean, rstd, out, p);
  else xcorr_fwd_kernel<false><<<grid, 256, 0, st>>>(x, w, bias, mean, rstd, out, p);
  HB_LAUNCH_CHECK();
  return 0;
}

// dw fp32 [Cout,Cin,KH,KW] (zeroed here) from g = d out fp32 [N,Cout,Ho,Wo]
int hb_xcorr2d_wgrad(const float* x, const float* w, const float* g, const float* mean, const float* rstd, float* dw,
                     int N, int Cin, int H, int W, int Cout, int KH, int KW, int stride, int pad, int dil, int mode,
                     int normalize, float eps, void* stream) {
  // grid: (K tiles, Cout tiles, splits over N*L)
  XcParams p;
  if (!make_params(p, N, Cin, H, W, Cout, KH, KW, stride, pad, dil, normalize, eps) || (Cout + TC - 1) / TC > 65535)
    return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(dw, 0, sizeof(float) * (size_t)Cout * p.K, st);
  if (e != cudaSuccess) return (int)e;
  const long long M = (long long)N * p.L;
  const long long chunks = (M + TL - 1) / TL;
  const int tiles = ((p.K + TK - 1) / TK) * ((Cout + TC - 1) / TC);
  long long splits = (HB_NUM_SMS * 2 + tiles - 1) / tiles;
  if (splits > chunks) splits = chunks;
  if (splits < 1) splits = 1;
  if (splits > 65535) splits = 65535;
  const int cps = (int)((chunks + splits - 1) / splits);
  dim3 grid((p.K + TK - 1) / TK, (Cout + TC - 1) / TC, (unsigned)((chunks + cps - 1) / cps));
  if (mode == 1) xcorr_wgrad_kernel<true><<<grid, 256, 0, st>>>(x, w, g, mean, rstd, dw, p, cps);
  else xcorr_wgrad_kernel<false><<<grid, 256, 0, st>>>(x, w, g, mean, rstd, dw, p, cps);
  HB_LAUNCH_CHECK();
  return 0;
}

// input gradient of add2d without slice normalisation (the only configuration in which the reference's own
// backward reaches x: with normalisation its in-place patch update makes autograd raise).
int hb_add2d_dgrad(const float* x, const float* w, const float* g, float* dx, int N, int Cin, int H, int W, int Cout,
                   int KH, int KW, int stride, int pad, int dil, void* stream) {
  XcParams p;
  if (!make_params(p, N, Cin, H, W, Cout, KH, KW, stride, pad, dil, 0, 0.f)) return (int)cudaErrorInvalidValue;
  const long long total = (long long)N * Cin * H * W;
  adder_dgrad_kernel<<<hb::stream_grid((size_t)total, 256), 256, 0, (cudaStream_t)stream>>>(x, w, g, dx, p);
  HB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
