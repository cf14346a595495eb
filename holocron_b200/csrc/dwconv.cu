// Depth-wise k x k convolution (groups == channels) over NHWC bf16 activations: forward, data gradient, weight/bias
// gradient. CUDA-core, HBM-bound (9 MAC per element for k = 3): every thread owns 8 consecutive channels
// (one 128-bit vector) of one output pixel; neighbouring threads share their taps through L1/L2.
// Used by FReLU (reference holocron/nn/modules/activation.py:58-82: conv k x k, groups = C, bias) and by the ReXNet
// blocks (reference holocron/models/classification/rexnet.py:112-125: dw 3x3, stride 1|2, no bias).
#include <cstdlib>
#include "common.cuh"

namespace {

using namespace hb;

constexpr int kThreads = 256;

// neighbouring threads re-read the same taps: the L1-allocating load
__device__ __forceinline__ void load8(const __nv_bfloat16* p, float* f) { unpack8(ld16(p), f); }

struct DwParams {
  int N, H, W, C, Ho, Wo, K, stride, pad;
};

// w: fp32 [C][K][K] (the nn.Conv2d weight [C,1,K,K]); bias fp32 [C] or null
__global__ void __launch_bounds__(kThreads) dw_fwd_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ w,
                                                          const float* __restrict__ bias, __nv_bfloat16* __restrict__ y,
                                                          DwParams p) {
  const int cv = p.C / 8;
  const long long total = (long long)p.N * p.Ho * p.Wo * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int cg = (int)(i % cv);
    long long t = i / cv;
    const int wo = (int)(t % p.Wo); t /= p.Wo;
    const int ho = (int)(t % p.Ho);
    const int n = (int)(t / p.Ho);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = bias ? bias[cg * 8 + j] : 0.f;
    for (int r = 0; r < p.K; ++r) {
      const int hi = ho * p.stride + r - p.pad;
      if (hi < 0 || hi >= p.H) continue;
      for (int s = 0; s < p.K; ++s) {
        const int wi = wo * p.stride + s - p.pad;
        if (wi < 0 || wi >= p.W) continue;
        float xv[8];
        load8(x + (((long long)n * p.H + hi) * p.W + wi) * p.C + cg * 8, xv);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = fmaf(xv[j], __ldg(w + ((cg * 8 + j) * p.K + r) * p.K + s), acc[j]);
      }
    }
    store8(y + i * 8, acc);
  }
}

// dx[n,h,w,c] = sum_{r,s} dy[n,(h+pad-r)/stride,(w+pad-s)/stride,c] * w[c,r,s]   (only exact divisions)
__global__ void __launch_bounds__(kThreads) dw_bwd_data_kernel(const __nv_bfloat16* __restrict__ dy,
                                                               const float* __restrict__ w,
                                                               __nv_bfloat16* __restrict__ dx, DwParams p) {
  const int cv = p.C / 8;
  const long long total = (long long)p.N * p.H * p.W * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int cg = (int)(i % cv);
    long long t = i / cv;
    const int wi = (int)(t % p.W); t /= p.W;
    const int hi = (int)(t % p.H);
    const int n = (int)(t / p.H);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int r = 0; r < p.K; ++r) {
      const int hn = hi + p.pad - r;
      if (hn < 0 || hn % p.stride != 0) continue;
      const int ho = hn / p.stride;
      if (ho >= p.Ho) continue;
      for (int s = 0; s < p.K; ++s) {
        const int wn = wi + p.pad - s;
        if (wn < 0 || wn % p.stride != 0) continue;
        const int wo = wn / p.stride;
        if (wo >= p.Wo) continue;
        float g[8];
        load8(dy + (((long long)n * p.Ho + ho) * p.Wo + wo) * p.C + cg * 8, g);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = fmaf(g[j], __ldg(w + ((cg * 8 + j) * p.K + r) * p.K + s), acc[j]);
      }
    }
    store8(dx + i * 8, acc);
  }
}

// ---- 3x3 specialisations: fixed channel group per thread (block = channel groups x pixel lanes, as in the BN
// kernels), the block's slab of the filter sits in shared memory (float4 reads). The generic kernels above
// re-read 72 scalar weights per output vector and recompute the channel group of every element: instruction-bound,
// far from the HBM time on the ReXNet expansions.
// kStride: 1 or 2 known at compile time (the backward index arithmetic divides by the stride: a runtime divisor costs
// ~40 instructions per tap, which makes the data-gradient pass instruction bound); 0 = runtime stride.
template <bool kBackward, int kStride>
__global__ void __launch_bounds__(kThreads, 3) dw3x3_kernel(const __nv_bfloat16* __restrict__ src, const float* __restrict__ w,
                                                         const float* __restrict__ bias, __nv_bfloat16* __restrict__ dst,
                                                         DwParams p, int cg_t, int rows_t) {
  // forward:  src = x [N,H,W,C],   dst = y  [N,Ho,Wo,C]: y[ho,wo]  = b + sum_{r,s} x[ho*st+r-pad, wo*st+s-pad] * w[r,s]
  // backward: src = dy [N,Ho,Wo,C], dst = dx [N,H,W,C]:  dx[hi,wi] = sum_{r,s} dy[(hi+pad-r)/st, (wi+pad-s)/st] * w[r,s]
  __shared__ __align__(16) float ws[9][256];   // the block's channel slab of the filter, tap-major
  const int cv = p.C / 8;
  const int tx = threadIdx.x % cg_t, ty = threadIdx.x / cg_t;
  const int cg = blockIdx.y * cg_t + tx;
  for (int i = threadIdx.x; i < 9 * cg_t * 8; i += kThreads) {
    const int k = i / (cg_t * 8), ch = i % (cg_t * 8);
    const int c = blockIdx.y * cg_t * 8 + ch;
    ws[k][ch] = c < p.C ? w[c * 9 + k] : 0.f;
  }
  __syncthreads();
  if (ty >= rows_t || cg >= cv) return;
  float b[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) b[j] = (!kBackward && bias) ? bias[cg * 8 + j] : 0.f;
  const int stride = kStride > 0 ? kStride : p.stride;
  const int OH = kBackward ? p.H : p.Ho, OW = kBackward ? p.W : p.Wo;   // grid walked by this kernel
  const int IH = kBackward ? p.Ho : p.H, IW = kBackward ? p.Wo : p.W;   // grid of src
  const long long M = (long long)p.N * OH * OW;
  const long long stride_m = (long long)gridDim.x * rows_t;
  for (long long m = (long long)blockIdx.x * rows_t + ty; m < M; m += stride_m) {
    // 32-bit index arithmetic (the launcher checks M < 2^31): 64-bit runtime divisions cost ~100 instructions each
    const unsigned mu = (unsigned)m;
    const unsigned t1 = mu / (unsigned)OW;
    const int ow = (int)(mu - t1 * (unsigned)OW);
    const long long n = t1 / (unsigned)OH;
    const int oh = (int)(t1 - (unsigned)n * (unsigned)OH);
    const __nv_bfloat16* sn = src + n * IH * IW * p.C + cg * 8;
    Vec16<__nv_bfloat16> v[9];
    bool ok[9];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
      for (int s2 = 0; s2 < 3; ++s2) {
        int ih, iw;
        bool good;
        if (!kBackward) {
          ih = oh * stride + r - p.pad; iw = ow * stride + s2 - p.pad;
          good = ih >= 0 && ih < IH && iw >= 0 && iw < IW;
        } else {
          const int hn = oh + p.pad - r, wn = ow + p.pad - s2;
          good = hn >= 0 && wn >= 0 && (stride == 1 || ((hn % stride) == 0 && (wn % stride) == 0));
          ih = hn / stride; iw = wn / stride;
          good = good && ih < IH && iw < IW;
        }
        ok[r * 3 + s2] = good;
        if (good) v[r * 3 + s2] = ld16(sn + ((long long)ih * IW + iw) * p.C);   // all 9 loads issued before the first use
      }
    }
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = b[j];
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      if (ok[k]) {
        const float4 w0 = *reinterpret_cast<const float4*>(&ws[k][tx * 8]);
        const float4 w1 = *reinterpret_cast<const float4*>(&ws[k][tx * 8 + 4]);
        const float wk[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = fmaf(__bfloat162float(v[k].v[j]), wk[j], acc[j]);
      }
    }
    store8(dst + m * p.C + cg * 8, acc);
  }
}

// ---- four horizontally adjacent outputs per thread ------------------------------------------------------------------
// The one-output-per-thread kernel above issues 9 vector loads, 72 converts, 18 shared-memory filter reads, two integer
// divisions and 9 bounds predicates per 8 output values and is instruction-bound on the ReXNet expansions. With 4 outputs of one row per thread the 3 input rows are loaded once
// (3 x (3*S+3) vectors for stride S instead of 36), the filter slab is read once per quad and the index arithmetic is
// amortised over 32 output values.
//   forward  (kFlip = 0): y[oh, ow]  = b + sum_{r,s} x[oh*S + r - pad, ow*S + s - pad] * w[r, s]
//   backward (kFlip = 1, S = 1 only): dx[h, w] = sum_{r,s} dy[h + pad - r, w + pad - s] * w[r, s]
//            = correlation of dy with the FLIPPED filter and padding 2 - pad
template <int kStride, bool kFlip>
__global__ void __launch_bounds__(kThreads, 2) dw3x3_quad_kernel(const __nv_bfloat16* __restrict__ src, const float* __restrict__ w,
                                                              const float* __restrict__ bias, __nv_bfloat16* __restrict__ dst,
                                                              int N, int IH, int IW, int OH, int OW, int C, int pad, int cg_t,
                                                              int rows_t) {
  __shared__ __align__(16) float ws[9][256];   // the block's channel slab of the filter, tap-major (flipped for kFlip)
  const int cv = C / 8;
  const int tx = threadIdx.x % cg_t, ty = threadIdx.x / cg_t;
  const int cg = blockIdx.y * cg_t + tx;
  for (int i = threadIdx.x; i < 9 * cg_t * 8; i += kThreads) {
    const int k = i / (cg_t * 8), ch = i % (cg_t * 8);
    const int c = blockIdx.y * cg_t * 8 + ch;
    ws[k][ch] = c < C ? w[c * 9 + (kFlip ? 8 - k : k)] : 0.f;
  }
  __syncthreads();
  if (ty >= rows_t || cg >= cv) return;
  float b[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) b[j] = (!kFlip && bias) ? bias[cg * 8 + j] : 0.f;
  constexpr int kIn = 3 * kStride + 3;          // input columns feeding 4 outputs: (4 - 1) * S + 3
  const int qw = (OW + 3) >> 2;                 // quads per output row
  const unsigned total = (unsigned)N * OH * qw;
  for (unsigned q = blockIdx.x * rows_t + ty; q < total; q += gridDim.x * rows_t) {
    const unsigned t1 = q / (unsigned)qw;
    const int ow0 = (int)(q - t1 * (unsigned)qw) * 4;
    const unsigned n = t1 / (unsigned)OH;
    const int oh = (int)(t1 - n * (unsigned)OH);
    const int iw0 = ow0 * kStride - pad;
    float acc[4][8];
#pragma unroll
    for (int o = 0; o < 4; ++o)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[o][j] = b[j];
    const __nv_bfloat16* sn = src + (size_t)n * IH * IW * C + cg * 8;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int ih = oh * kStride + r - pad;
      if (ih < 0 || ih >= IH) continue;
      const __nv_bfloat16* row = sn + (size_t)ih * IW * C;
      Vec16<__nv_bfloat16> v[kIn];
#pragma unroll
      for (int c = 0; c < kIn; ++c) {           // all loads of the row in flight before the first use
        const int iw = iw0 + c;
        if (iw >= 0 && iw < IW) v[c] = ld16(row + (size_t)iw * C);
        else v[c].raw = make_uint4(0, 0, 0, 0);
      }
      float wk[3][8];
#pragma unroll
      for (int s2 = 0; s2 < 3; ++s2) {
        const float4 w0 = *reinterpret_cast<const float4*>(&ws[r * 3 + s2][tx * 8]);
        const float4 w1 = *reinterpret_cast<const float4*>(&ws[r * 3 + s2][tx * 8 + 4]);
        wk[s2][0] = w0.x; wk[s2][1] = w0.y; wk[s2][2] = w0.z; wk[s2][3] = w0.w;
        wk[s2][4] = w1.x; wk[s2][5] = w1.y; wk[s2][6] = w1.z; wk[s2][7] = w1.w;
      }
#pragma unroll
      for (int c = 0; c < kIn; ++c) {
        float f[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] = __bfloat162float(v[c].v[j]);
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          const int s2 = c - o * kStride;        // compile-time after unrolling
          if (s2 >= 0 && s2 < 3) {
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[o][j] = fmaf(f[j], wk[s2][j], acc[o][j]);
          }
        }
      }
    }
    __nv_bfloat16* out = dst + (((size_t)n * OH + oh) * OW + ow0) * C + cg * 8;
#pragma unroll
    for (int o = 0; o < 4; ++o)
      if (ow0 + o < OW) store8(out + (size_t)o * C, acc[o]);
  }
}

// Stride-2, pad-1 data gradient, four consecutive dx columns (w0 % 4 == 0) per thread. With stride 2 only the taps whose
// parity matches reach a dx pixel: row h takes filter row 1 (h even, dy row h/2) or rows 0 and 2 (h odd, dy rows (h+1)/2 and
// (h-1)/2); along W the quad {w0..w0+3} reads the three dy columns c0 = w0/2, c0+1, c0+2 in a fixed pattern:
//   dx[w0]   += dy[c0]   w[.,1]              dx[w0+1] += dy[c0+1] w[.,0] + dy[c0]   w[.,2]
//   dx[w0+2] += dy[c0+1] w[.,1]              dx[w0+3] += dy[c0+2] w[.,0] + dy[c0+1] w[.,2]
// 3 - 6 vector loads per 4 outputs; the one-output kernel issues 9 predicated loads per output.
__global__ void __launch_bounds__(kThreads, 2) dw3x3_dgrad_s2_quad_kernel(const __nv_bfloat16* __restrict__ dy,
                                                                        const float* __restrict__ w, __nv_bfloat16* __restrict__ dx,
                                                                        int N, int H, int W, int Ho, int Wo, int C, int cg_t,
                                                                        int rows_t) {
  __shared__ __align__(16) float ws[9][256];
  const int cv = C / 8;
  const int tx = threadIdx.x % cg_t, ty = threadIdx.x / cg_t;
  const int cg = blockIdx.y * cg_t + tx;
  for (int i = threadIdx.x; i < 9 * cg_t * 8; i += kThreads) {
    const int k = i / (cg_t * 8), ch = i % (cg_t * 8);
    const int c = blockIdx.y * cg_t * 8 + ch;
    ws[k][ch] = c < C ? w[c * 9 + k] : 0.f;
  }
  __syncthreads();
  if (ty >= rows_t || cg >= cv) return;
  const int qw = (W + 3) >> 2;
  const unsigned total = (unsigned)N * H * qw;
  for (unsigned q = blockIdx.x * rows_t + ty; q < total; q += gridDim.x * rows_t) {
    const unsigned t1 = q / (unsigned)qw;
    const int w0 = (int)(q - t1 * (unsigned)qw) * 4;
    const unsigned n = t1 / (unsigned)H;
    const int h = (int)(t1 - n * (unsigned)H);
    const int c0 = w0 >> 1;
    float acc[4][8];
#pragma unroll
    for (int o = 0; o < 4; ++o)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[o][j] = 0.f;
    const __nv_bfloat16* dn = dy + (size_t)n * Ho * Wo * C + cg * 8;
    for (int r = (h & 1) ? 0 : 1; r < 3; r += 2) {
      const int oh = (h + 1 - r) >> 1;
      if (oh >= Ho) continue;
      const __nv_bfloat16* row = dn + (size_t)oh * Wo * C;
      Vec16<__nv_bfloat16> v[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        if (c0 + i < Wo) v[i] = ld16(row + (size_t)(c0 + i) * C);
        else v[i].raw = make_uint4(0, 0, 0, 0);
      }
      float wk[3][8];
#pragma unroll
      for (int s2 = 0; s2 < 3; ++s2) {
        const float4 a = *reinterpret_cast<const float4*>(&ws[r * 3 + s2][tx * 8]);
        const float4 b = *reinterpret_cast<const float4*>(&ws[r * 3 + s2][tx * 8 + 4]);
        wk[s2][0] = a.x; wk[s2][1] = a.y; wk[s2][2] = a.z; wk[s2][3] = a.w;
        wk[s2][4] = b.x; wk[s2][5] = b.y; wk[s2][6] = b.z; wk[s2][7] = b.w;
      }
      float f[3][8];
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) f[i][j] = __bfloat162float(v[i].v[j]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        acc[0][j] = fmaf(f[0][j], wk[1][j], acc[0][j]);
        acc[1][j] = fmaf(f[1][j], wk[0][j], fmaf(f[0][j], wk[2][j], acc[1][j]));
        acc[2][j] = fmaf(f[1][j], wk[1][j], acc[2][j]);
        acc[3][j] = fmaf(f[2][j], wk[0][j], fmaf(f[1][j], wk[2][j], acc[3][j]));
      }
    }
    __nv_bfloat16* out = dx + (((size_t)n * H + h) * W + w0) * C + cg * 8;
#pragma unroll
    for (int o = 0; o < 4; ++o)
      if (w0 + o < W) store8(out + (size_t)o * C, acc[o]);
  }
}

inline dim3 dw_quad_grid(long long quads, int cv, int& cg_t, int& rows_t, int per_sm) {
  const int nslab = (cv + 31) / 32;
  cg_t = (cv + nslab - 1) / nslab;
  rows_t = kThreads / cg_t;
  const int slabs = (cv + cg_t - 1) / cg_t;
  long long gx = (quads + rows_t * 2 - 1) / (rows_t * 2);
  long long cap = (HB_NUM_SMS * per_sm) / slabs;
  if (cap < 1) cap = 1;
  if (gx > cap) gx = cap;
  if (gx < 1) gx = 1;
  return dim3((unsigned)gx, (unsigned)slabs);
}

inline dim3 dw_grid(long long M, int cv, int& cg_t, int& rows_t, int per_sm) {
  const int nslab = (cv + 31) / 32;
  cg_t = (cv + nslab - 1) / nslab;      // balanced channel slabs (see bn_act.cu)
  rows_t = kThreads / cg_t;
  const int slabs = (cv + cg_t - 1) / cg_t;
  long long gx = (M + rows_t * 4 - 1) / (rows_t * 4);
  long long cap = (HB_NUM_SMS * per_sm) / slabs;
  if (cap < 1) cap = 1;
  if (gx > cap) gx = cap;
  if (gx < 1) gx = 1;
  return dim3((unsigned)gx, (unsigned)slabs);
}

// dw[c,r,s] = sum_{n,ho,wo} dy * x_shifted ; db[c] = sum dy.  part: double [gridDim.x][C][KK+1] per-block partial sums (last
// column = bias grad), folded in a fixed order by dw_weight_finalize_kernel: deterministic (the first version added doubles
// atomically). Block geometry as in the BN kernels: tx = channel group within a 32-group slab, ty = pixel lane
template <int KS>
__global__ void __launch_bounds__(kThreads, KS == 3 ? 2 : 1) dw_bwd_weight_kernel(const __nv_bfloat16* __restrict__ x,
                                                                 const __nv_bfloat16* __restrict__ dy, double* part,
                                                                 DwParams p, int cg_t, int rows_t) {
  constexpr int KK = KS * KS;
  __shared__ float red[kThreads * 8];
  const int cv = p.C / 8;
  const int tx = threadIdx.x % cg_t, ty = threadIdx.x / cg_t;
  const int cg = blockIdx.y * cg_t + tx;
  const bool active = ty < rows_t && cg < cv;
  float acc[KK + 1][8];
#pragma unroll
  for (int k = 0; k <= KK; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[k][j] = 0.f;
  if (active) {
    const long long M = (long long)p.N * p.Ho * p.Wo;
    const long long stride_m = (long long)gridDim.x * rows_t;
    for (long long m = (long long)blockIdx.x * rows_t + ty; m < M; m += stride_m) {
      const unsigned mu = (unsigned)m;            // M < 2^31 checked by the launcher
      const unsigned t1 = mu / (unsigned)p.Wo;
      const int wo = (int)(mu - t1 * (unsigned)p.Wo);
      const int n = (int)(t1 / (unsigned)p.Ho);
      const int ho = (int)(t1 - (unsigned)n * (unsigned)p.Ho);
      float g[8];
      if constexpr (KS == 3) {
        // loads are issued one filter row (3 taps) ahead of their use: 80 accumulators leave no room for all 9 vectors
        Vec16<__nv_bfloat16> gv = ld16(dy + m * p.C + cg * 8);
#pragma unroll
        for (int j = 0; j < 8; ++j) { g[j] = __bfloat162float(gv.v[j]); acc[KK][j] += g[j]; }
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const int hi = ho * p.stride + r - p.pad;
          const bool hok = hi >= 0 && hi < p.H;
          Vec16<__nv_bfloat16> xv3[3];
          bool ok[3];
#pragma unroll
          for (int s = 0; s < 3; ++s) {
            const int wi = wo * p.stride + s - p.pad;
            ok[s] = hok && wi >= 0 && wi < p.W;
            if (ok[s]) xv3[s] = ld16(x + (((long long)n * p.H + hi) * p.W + wi) * p.C + cg * 8);
          }
#pragma unroll
          for (int s = 0; s < 3; ++s) {
            if (ok[s]) {
#pragma unroll
              for (int j = 0; j < 8; ++j) acc[r * 3 + s][j] = fmaf(g[j], __bfloat162float(xv3[s].v[j]), acc[r * 3 + s][j]);
            }
          }
        }
        continue;
      }
      load8(dy + m * p.C + cg * 8, g);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[KK][j] += g[j];
#pragma unroll
      for (int r = 0; r < KS; ++r) {
        const int hi = ho * p.stride + r - p.pad;
        if (hi < 0 || hi >= p.H) continue;
#pragma unroll
        for (int s = 0; s < KS; ++s) {
          const int wi = wo * p.stride + s - p.pad;
          if (wi < 0 || wi >= p.W) continue;
          float xv[8];
          load8(x + (((long long)n * p.H + hi) * p.W + wi) * p.C + cg * 8, xv);
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[r * KS + s][j] = fmaf(g[j], xv[j], acc[r * KS + s][j]);
        }
      }
    }
  }
  const int nch = cg_t * 8;
#pragma unroll
  for (int k = 0; k <= KK; ++k) {
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) red[threadIdx.x * 8 + j] = acc[k][j];
    __syncthreads();
    for (int ch = threadIdx.x; ch < nch; ch += kThreads) {
      const int ctx = ch / 8, j = ch % 8;
      const int gcg = blockIdx.y * cg_t + ctx;
      if (gcg >= cv) continue;
      double a = 0.0;
      for (int r = 0; r < rows_t; ++r) a += (double)red[(r * cg_t + ctx) * 8 + j];
      part[((size_t)blockIdx.x * p.C + gcg * 8 + j) * (KK + 1) + k] = a;
    }
  }
}

// 3x3 weight gradient, stride 1 / 2: a thread owns ONE filter row r and FOUR consecutive output pixels of a row. It loads the 4
// dy vectors and the 3*S + 3 input vectors of input row oh*S + r - pad (all in flight before the first use) and keeps 3 taps x 8
// channels (+ the bias column on r == 0) of accumulators: 32 instead of 80, so two blocks per SM fit without serialising the
// loads filter row by filter row, and 7.5 / 11.25 vector loads per output pixel instead of 10. ty = lane * 3 + r.
template <int kStride>
__global__ void __launch_bounds__(kThreads, 2) dw3x3_wgrad_quad_kernel(const __nv_bfloat16* __restrict__ x,
                                                                    const __nv_bfloat16* __restrict__ dy, double* part,
                                                                    DwParams p, int cg_t, int lanes) {
  __shared__ float red[kThreads * 8];
  const int cv = p.C / 8;
  const int tx = threadIdx.x % cg_t, ty = threadIdx.x / cg_t;
  const int r = ty % 3, lane = ty / 3;
  const int cg = blockIdx.y * cg_t + tx;
  const bool active = lane < lanes && cg < cv;
  float acc[4][8];
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[k][j] = 0.f;
  if (active) {
    constexpr int kIn = 3 * kStride + 3;
    const int qw = (p.Wo + 3) >> 2;
    const unsigned total = (unsigned)p.N * p.Ho * qw;
    const size_t C = (size_t)p.C;
    for (unsigned q = blockIdx.x * lanes + lane; q < total; q += gridDim.x * lanes) {
      const unsigned t1 = q / (unsigned)qw;
      const int ow0 = (int)(q - t1 * (unsigned)qw) * 4;
      const unsigned n = t1 / (unsigned)p.Ho;
      const int oh = (int)(t1 - n * (unsigned)p.Ho);
      const int ih = oh * kStride + r - p.pad;
      const bool hok = ih >= 0 && ih < p.H;
      if (!hok && r != 0) continue;
      const __nv_bfloat16* dyp = dy + (((size_t)n * p.Ho + oh) * p.Wo + ow0) * C + cg * 8;
      Vec16<__nv_bfloat16> gv[4], xv[kIn];
#pragma unroll
      for (int o = 0; o < 4; ++o) {
        if (ow0 + o < p.Wo) gv[o] = ld16(dyp + (size_t)o * C);
        else gv[o].raw = make_uint4(0, 0, 0, 0);
      }
      if (hok) {
        const __nv_bfloat16* row = x + (((size_t)n * p.H + ih) * p.W) * C + cg * 8;
        const int iw0 = ow0 * kStride - p.pad;
#pragma unroll
        for (int c = 0; c < kIn; ++c) {
          const int iw = iw0 + c;
          if (iw >= 0 && iw < p.W) xv[c] = ld16(row + (size_t)iw * C);
          else xv[c].raw = make_uint4(0, 0, 0, 0);
        }
      }
      float g[4][8];
#pragma unroll
      for (int o = 0; o < 4; ++o)
#pragma unroll
        for (int j = 0; j < 8; ++j) g[o][j] = __bfloat162float(gv[o].v[j]);
      if (r == 0) {
#pragma unroll
        for (int o = 0; o < 4; ++o)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[3][j] += g[o][j];
      }
      if (hok) {
#pragma unroll
        for (int c = 0; c < kIn; ++c) {
          float f[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) f[j] = __bfloat162float(xv[c].v[j]);
#pragma unroll
          for (int o = 0; o < 4; ++o) {
            const int s2 = c - o * kStride;   // compile-time after unrolling
            if (s2 >= 0 && s2 < 3) {
#pragma unroll
              for (int j = 0; j < 8; ++j) acc[s2][j] = fmaf(g[o][j], f[j], acc[s2][j]);
            }
          }
        }
      }
    }
  }
  const int nch = cg_t * 8;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) red[threadIdx.x * 8 + j] = acc[k][j];
    __syncthreads();
    const int nr = k < 3 ? 3 : 1;             // the bias column lives on the r == 0 threads only
    for (int idx = threadIdx.x; idx < nch * nr; idx += kThreads) {
      const int rr = idx / nch, ch = idx - rr * nch;
      const int ctx = ch / 8, j = ch % 8;
      const int gcg = blockIdx.y * cg_t + ctx;
      if (gcg >= cv) continue;
      double a = 0.0;
      for (int l = 0; l < lanes; ++l) a += (double)red[(((l * 3 + rr) * cg_t) + ctx) * 8 + j];
      part[((size_t)blockIdx.x * p.C + gcg * 8 + j) * 10 + (k < 3 ? rr * 3 + k : 9)] = a;
    }
  }
}

// dw / db = sum over the gx row blocks of part[g][c][k]: block = 8 entries (one 64-byte run) x 32 block lanes, four rows in
// flight, lane sums combined in lane order (fixed order, see bn_finalize_kernel)
__global__ void __launch_bounds__(256) dw_weight_finalize_kernel(const double* part, int gx, float* dw, float* db, int C, int KK) {
  __shared__ double red[32][8];
  const int E = C * (KK + 1);
  const int i = blockIdx.x * 8 + threadIdx.x;
  double a = 0.0;
  if (i < E) {
    int g = threadIdx.y;
    for (; g + 96 < gx; g += 128) {
      double v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = part[(size_t)(g + 32 * u) * E + i];
#pragma unroll
      for (int u = 0; u < 4; ++u) a += v[u];
    }
    for (; g < gx; g += 32) a += part[(size_t)g * E + i];
  }
  red[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.y != 0 || i >= E) return;
  a = 0.0;
#pragma unroll
  for (int l = 0; l < 32; ++l) a += red[l][threadIdx.x];
  const int c = i / (KK + 1), k = i % (KK + 1);
  if (k < KK) dw[c * KK + k] = (float)a;
  else if (db) db[c] = (float)a;
}

// channel-slab geometry of the weight-gradient kernels and the number of row blocks (<= 2 blocks per SM over all slabs)
inline void dw_wgrad_geo(int C, int& cg_t, int& rows_t, int& slabs, int& gx_max) {
  const int cv = C / 8;
  const int nslab = (cv + 31) / 32;
  cg_t = (cv + nslab - 1) / nslab;
  rows_t = kThreads / cg_t;
  slabs = (cv + cg_t - 1) / cg_t;
  gx_max = (HB_NUM_SMS * 2) / slabs;
  if (gx_max < 1) gx_max = 1;
}

// 0 when the geometry is supported (fills p), otherwise cudaErrorInvalidValue, before any launch or device query:
// N, H, W, C, K, stride >= 1, pad >= 0, C % 8 == 0 and a filter that fits the padded input (Ho, Wo >= 1). Integer
// division truncates towards zero, so H + 2 * pad - K is checked for a negative value itself: (H + 2 * pad - K) / stride + 1
// alone gives Ho = 1 for a filter up to stride - 1 pixels too large.
int make_params(DwParams& p, int N, int H, int W, int C, int K, int stride, int pad) {
  if (N < 1 || H < 1 || W < 1 || C < 1 || C % 8 != 0 || K < 1 || stride < 1 || pad < 0) return (int)cudaErrorInvalidValue;
  const long long h = (long long)H + 2LL * pad - K, w = (long long)W + 2LL * pad - K;
  if (h < 0 || w < 0 || h / stride >= 0x7fffffffLL || w / stride >= 0x7fffffffLL) return (int)cudaErrorInvalidValue;
  p = DwParams{N, H, W, C, (int)(h / stride + 1), (int)(w / stride + 1), K, stride, pad};
  return 0;
}

}  // namespace

extern "C" {

// y[N,Ho,Wo,C] = dwconv(x[N,H,W,C], w fp32 [C,K,K]) + bias; C % 8 == 0
int hb_dwconv_fwd_bf16(const void* x, const float* w, const float* bias, void* y, int N, int H, int W, int C, int K,
                       int stride, int pad, void* stream) {
  DwParams p;
  if (int rc = make_params(p, N, H, W, C, K, stride, pad)) return rc;
  const long long total = (long long)N * p.Ho * p.Wo * (C / 8);
  if (K == 3 && (long long)N * p.Ho * p.Wo < 0x7fffffffLL) {
    int cg_t, rows_t;
    const __nv_bfloat16* xb = (const __nv_bfloat16*)x;
    __nv_bfloat16* yb = (__nv_bfloat16*)y;
    cudaStream_t st = (cudaStream_t)stream;
    static const bool quad_on = getenv("HB_DISABLE_DW_QUAD") == nullptr;
    if (quad_on && (stride == 1 || stride == 2) && p.Wo >= 4) {
      const long long quads = (long long)N * p.Ho * ((p.Wo + 3) / 4);
      const dim3 qgrid = dw_quad_grid(quads, C / 8, cg_t, rows_t, 2);
      if (stride == 1) dw3x3_quad_kernel<1, false><<<qgrid, kThreads, 0, st>>>(xb, w, bias, yb, N, H, W, p.Ho, p.Wo, C, pad, cg_t, rows_t);
      else dw3x3_quad_kernel<2, false><<<qgrid, kThreads, 0, st>>>(xb, w, bias, yb, N, H, W, p.Ho, p.Wo, C, pad, cg_t, rows_t);
      HB_LAUNCH_CHECK();
      return 0;
    }
    const dim3 grid = dw_grid((long long)N * p.Ho * p.Wo, C / 8, cg_t, rows_t, 3);
    if (stride == 1) dw3x3_kernel<false, 1><<<grid, kThreads, 0, st>>>(xb, w, bias, yb, p, cg_t, rows_t);
    else if (stride == 2) dw3x3_kernel<false, 2><<<grid, kThreads, 0, st>>>(xb, w, bias, yb, p, cg_t, rows_t);
    else dw3x3_kernel<false, 0><<<grid, kThreads, 0, st>>>(xb, w, bias, yb, p, cg_t, rows_t);
    HB_LAUNCH_CHECK();
    return 0;
  }
  dw_fwd_kernel<<<stream_grid((size_t)total, kThreads, 16), kThreads, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x, w, bias, (__nv_bfloat16*)y, p);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_dwconv_bwd_data_bf16(const void* dy, const float* w, void* dx, int N, int H, int W, int C, int K, int stride,
                            int pad, void* stream) {
  DwParams p;
  if (int rc = make_params(p, N, H, W, C, K, stride, pad)) return rc;
  const long long total = (long long)N * H * W * (C / 8);
  if (K == 3 && (long long)N * H * W < 0x7fffffffLL) {
    int cg_t, rows_t;
    const __nv_bfloat16* dyb = (const __nv_bfloat16*)dy;
    __nv_bfloat16* dxb = (__nv_bfloat16*)dx;
    cudaStream_t st = (cudaStream_t)stream;
    static const bool quad_on = getenv("HB_DISABLE_DW_QUAD") == nullptr;
    if (quad_on && stride == 1 && W >= 4 && pad <= 2) {
      // stride 1: the data gradient is the correlation of dy [N,Ho,Wo,C] with the flipped filter, padding 2 - pad
      const long long quads = (long long)N * H * ((W + 3) / 4);
      const dim3 qgrid = dw_quad_grid(quads, C / 8, cg_t, rows_t, 2);
      dw3x3_quad_kernel<1, true><<<qgrid, kThreads, 0, st>>>(dyb, w, nullptr, dxb, N, p.Ho, p.Wo, H, W, C, 2 - pad, cg_t, rows_t);
      HB_LAUNCH_CHECK();
      return 0;
    }
    if (quad_on && stride == 2 && pad == 1 && W >= 4) {
      const long long quads = (long long)N * H * ((W + 3) / 4);
      const dim3 qgrid = dw_quad_grid(quads, C / 8, cg_t, rows_t, 2);
      dw3x3_dgrad_s2_quad_kernel<<<qgrid, kThreads, 0, st>>>(dyb, w, dxb, N, H, W, p.Ho, p.Wo, C, cg_t, rows_t);
      HB_LAUNCH_CHECK();
      return 0;
    }
    const dim3 grid = dw_grid((long long)N * H * W, C / 8, cg_t, rows_t, 3);
    if (stride == 1) dw3x3_kernel<true, 1><<<grid, kThreads, 0, st>>>(dyb, w, nullptr, dxb, p, cg_t, rows_t);
    else if (stride == 2) dw3x3_kernel<true, 2><<<grid, kThreads, 0, st>>>(dyb, w, nullptr, dxb, p, cg_t, rows_t);
    else dw3x3_kernel<true, 0><<<grid, kThreads, 0, st>>>(dyb, w, nullptr, dxb, p, cg_t, rows_t);
    HB_LAUNCH_CHECK();
    return 0;
  }
  dw_bwd_data_kernel<<<stream_grid((size_t)total, kThreads, 16), kThreads, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)dy, w, (__nv_bfloat16*)dx, p);
  HB_LAUNCH_CHECK();
  return 0;
}

// doubles of scratch hb_dwconv_bwd_weight_bf16 needs for C channels and a K x K filter (per-block partial sums); 0 for
// the shapes it refuses (K outside {1, 3, 5, 7})
size_t hb_dwconv_wgrad_scratch_doubles(int C, int K) {
  if (C <= 0 || C % 8 != 0 || (K != 1 && K != 3 && K != 5 && K != 7)) return 0;
  int cg_t, rows_t, slabs, gx_max;
  dw_wgrad_geo(C, cg_t, rows_t, slabs, gx_max);
  return (size_t)gx_max * C * (K * K + 1);
}

// dw fp32 [C,K,K], db fp32 [C] (or NULL); scratch: double[hb_dwconv_wgrad_scratch_doubles(C, K)]. K in {1, 3, 5, 7}.
int hb_dwconv_bwd_weight_bf16(const void* x, const void* dy, float* dw, float* db, double* scratch, int N, int H, int W,
                              int C, int K, int stride, int pad, void* stream) {
  DwParams p;
  if (int rc = make_params(p, N, H, W, C, K, stride, pad)) return rc;
  if (K != 1 && K != 3 && K != 5 && K != 7) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  const int KK = K * K;
  int cg_t, rows_t, slabs, gx_max;
  dw_wgrad_geo(C, cg_t, rows_t, slabs, gx_max);
  const long long M = (long long)N * p.Ho * p.Wo;
  if (M >= 0x7fffffffLL) return (int)cudaErrorInvalidValue;
  const __nv_bfloat16* xb = (const __nv_bfloat16*)x;
  const __nv_bfloat16* dyb = (const __nv_bfloat16*)dy;
  static const bool quad_on = getenv("HB_DISABLE_DW_QUAD") == nullptr;
  long long gx;
  if (quad_on && K == 3 && (stride == 1 || stride == 2) && rows_t >= 3) {
    const int lanes = rows_t / 3;
    const long long quads = (long long)N * p.Ho * ((p.Wo + 3) / 4);
    gx = (quads + lanes * 2 - 1) / (lanes * 2);
    if (gx > gx_max) gx = gx_max;
    if (gx < 1) gx = 1;
    const dim3 grid((unsigned)gx, (unsigned)slabs);
    if (stride == 1) dw3x3_wgrad_quad_kernel<1><<<grid, kThreads, 0, st>>>(xb, dyb, scratch, p, cg_t, lanes);
    else dw3x3_wgrad_quad_kernel<2><<<grid, kThreads, 0, st>>>(xb, dyb, scratch, p, cg_t, lanes);
  } else {
    gx = (M + rows_t * 8 - 1) / (rows_t * 8);
    if (gx > gx_max) gx = gx_max;
    if (gx < 1) gx = 1;
    const dim3 grid((unsigned)gx, (unsigned)slabs);
    switch (K) {
      case 1: dw_bwd_weight_kernel<1><<<grid, kThreads, 0, st>>>(xb, dyb, scratch, p, cg_t, rows_t); break;
      case 3: dw_bwd_weight_kernel<3><<<grid, kThreads, 0, st>>>(xb, dyb, scratch, p, cg_t, rows_t); break;
      case 5: dw_bwd_weight_kernel<5><<<grid, kThreads, 0, st>>>(xb, dyb, scratch, p, cg_t, rows_t); break;
      case 7: dw_bwd_weight_kernel<7><<<grid, kThreads, 0, st>>>(xb, dyb, scratch, p, cg_t, rows_t); break;
      default: return (int)cudaErrorInvalidValue;
    }
  }
  HB_LAUNCH_CHECK();
  dw_weight_finalize_kernel<<<(C * (KK + 1) + 7) / 8, dim3(8, 32), 0, st>>>(scratch, (int)gx, dw, db, C, KK);
  HB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
