// Depth-wise k x k convolution (groups == channels) over NHWC bf16 activations: forward, data gradient, weight/bias
// gradient. CUDA-core, HBM-bound (9 MAC per element for k = 3): every thread owns 8 consecutive channels
// (one 128-bit vector) of one output pixel; neighbouring threads share their taps through L1/L2.
// Used by FReLU (reference holocron/nn/modules/activation.py:58-82: conv k x k, groups = C, bias) and by the ReXNet
// blocks (reference holocron/models/classification/rexnet.py:112-125: dw 3x3, stride 1|2, no bias).
#include <cstdlib>
#include "common.cuh"
#include "slab.cuh"

namespace {

using namespace hb;

constexpr int kThreads = kSlabThreads;

// neighbouring threads re-read the same taps: the L1-allocating load
__device__ __forceinline__ void load8(const __nv_bfloat16* p, float* f) { unpack8(ld16(p), f); }

// the vector at p when ok, else zeros (p is then not read)
__device__ __forceinline__ Vec16<__nv_bfloat16> ld16_or_zero(const __nv_bfloat16* p, bool ok) {
  Vec16<__nv_bfloat16> v;
  if (ok) v = ld16(p);
  else v.raw = make_uint4(0, 0, 0, 0);
  return v;
}

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

// ---- 3x3 specialisations: fixed channel group per thread (block = channel groups x pixel lanes, the SlabGeo of
// slab.cuh), the block's slab of the filter sits in shared memory (float4 reads). The generic kernels above
// re-read 72 scalar weights per output vector and recompute the channel group of every element: instruction-bound,
// far from the HBM time on the ReXNet expansions. The slab kernels read the geometry as a __grid_constant__ parameter:
// passed as a plain by-value struct, ptxas spills dw3x3_kernel<false, 0>, which has no register to spare at 3 blocks/SM.

// The block's channel slab of the 3x3 filter w [C][9], tap-major: ws[k][ch] = w[slab channel ch][k], or tap 8 - k with
// kFlip; 0 past the last channel. Ends on a barrier, which every thread of the block has to reach.
template <bool kFlip>
__device__ __forceinline__ void stage_filter(float (&ws)[9][256], const float* __restrict__ w, const SlabGeo& g) {
  const int nch = g.cg_t * 8;
  for (int i = threadIdx.x; i < 9 * nch; i += kThreads) {
    const int k = i / nch, ch = i % nch;
    const int c = blockIdx.y * nch + ch;
    ws[k][ch] = c < g.cg_total * 8 ? w[c * 9 + (kFlip ? 8 - k : k)] : 0.f;
  }
  __syncthreads();
}

// the 8 staged filter values of tap k for channel group tx of the slab
__device__ __forceinline__ void tap8(const float (&ws)[9][256], int k, int tx, float* wk) {
  const float4 a = *reinterpret_cast<const float4*>(&ws[k][tx * 8]);
  const float4 b = *reinterpret_cast<const float4*>(&ws[k][tx * 8 + 4]);
  wk[0] = a.x; wk[1] = a.y; wk[2] = a.z; wk[3] = a.w;
  wk[4] = b.x; wk[5] = b.y; wk[6] = b.z; wk[7] = b.w;
}

// kStride: 1 or 2 known at compile time (the backward index arithmetic divides by the stride: a runtime divisor costs
// ~40 instructions per tap, which makes the data-gradient pass instruction bound); 0 = runtime stride.
template <bool kBackward, int kStride>
__global__ void __launch_bounds__(kThreads, 3) dw3x3_kernel(const __nv_bfloat16* __restrict__ src, const float* __restrict__ w,
                                                         const float* __restrict__ bias, __nv_bfloat16* __restrict__ dst,
                                                         DwParams p, const __grid_constant__ SlabGeo g) {
  // forward:  src = x [N,H,W,C],   dst = y  [N,Ho,Wo,C]: y[ho,wo]  = b + sum_{r,s} x[ho*st+r-pad, wo*st+s-pad] * w[r,s]
  // backward: src = dy [N,Ho,Wo,C], dst = dx [N,H,W,C]:  dx[hi,wi] = sum_{r,s} dy[(hi+pad-r)/st, (wi+pad-s)/st] * w[r,s]
  __shared__ __align__(16) float ws[9][256];
  const auto [tx, ty, cg, active] = g.thread();
  stage_filter<false>(ws, w, g);
  if (!active) return;
  float b[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) b[j] = (!kBackward && bias) ? bias[cg * 8 + j] : 0.f;
  const int stride = kStride > 0 ? kStride : p.stride;
  const int OH = kBackward ? p.H : p.Ho, OW = kBackward ? p.W : p.Wo;   // grid walked by this kernel
  const int IH = kBackward ? p.Ho : p.H, IW = kBackward ? p.Wo : p.W;   // grid of src
  const long long M = (long long)p.N * OH * OW;
  const long long stride_m = (long long)gridDim.x * g.rows_t;
  for (long long m = (long long)blockIdx.x * g.rows_t + ty; m < M; m += stride_m) {
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
        float wk[8];
        tap8(ws, k, tx, wk);
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
                                                              int N, int IH, int IW, int OH, int OW, int C, int pad,
                                                              const __grid_constant__ SlabGeo g) {
  __shared__ __align__(16) float ws[9][256];
  const auto [tx, ty, cg, active] = g.thread();
  stage_filter<kFlip>(ws, w, g);
  if (!active) return;
  float b[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) b[j] = (!kFlip && bias) ? bias[cg * 8 + j] : 0.f;
  constexpr int kIn = 3 * kStride + 3;          // input columns feeding 4 outputs: (4 - 1) * S + 3
  const int qw = (OW + 3) >> 2;                 // quads per output row
  const unsigned total = (unsigned)N * OH * qw;
  for (unsigned q = blockIdx.x * g.rows_t + ty; q < total; q += gridDim.x * g.rows_t) {
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
        v[c] = ld16_or_zero(row + (size_t)iw * C, iw >= 0 && iw < IW);
      }
      float wk[3][8];
#pragma unroll
      for (int s2 = 0; s2 < 3; ++s2) tap8(ws, r * 3 + s2, tx, wk[s2]);
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
                                                                        int N, int H, int W, int Ho, int Wo, int C,
                                                                        const __grid_constant__ SlabGeo g) {
  __shared__ __align__(16) float ws[9][256];
  const auto [tx, ty, cg, active] = g.thread();
  stage_filter<false>(ws, w, g);
  if (!active) return;
  const int qw = (W + 3) >> 2;
  const unsigned total = (unsigned)N * H * qw;
  for (unsigned q = blockIdx.x * g.rows_t + ty; q < total; q += gridDim.x * g.rows_t) {
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
      for (int i = 0; i < 3; ++i) v[i] = ld16_or_zero(row + (size_t)(c0 + i) * C, c0 + i < Wo);
      float wk[3][8];
#pragma unroll
      for (int s2 = 0; s2 < 3; ++s2) tap8(ws, r * 3 + s2, tx, wk[s2]);
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

// dw[c,r,s] = sum_{n,ho,wo} dy * x_shifted ; db[c] = sum dy.  part: double [gridDim.x][C][KK+1] per-block partial sums (last
// column = bias grad), folded in a fixed order by dw_weight_finalize_kernel: deterministic (the first version added doubles
// atomically). tx = channel group within the slab, ty = pixel lane (SlabGeo::thread)
template <int KS>
__global__ void __launch_bounds__(kThreads, KS == 3 ? 2 : 1) dw_bwd_weight_kernel(const __nv_bfloat16* __restrict__ x,
                                                                 const __nv_bfloat16* __restrict__ dy, double* part,
                                                                 DwParams p, const __grid_constant__ SlabGeo g) {
  constexpr int KK = KS * KS;
  __shared__ float red[kThreads * 8];
  const auto [tx, ty, cg, active] = g.thread();
  float acc[KK + 1][8];
#pragma unroll
  for (int k = 0; k <= KK; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[k][j] = 0.f;
  if (active) {
    const long long M = (long long)p.N * p.Ho * p.Wo;
    const long long stride_m = (long long)gridDim.x * g.rows_t;
    for (long long m = (long long)blockIdx.x * g.rows_t + ty; m < M; m += stride_m) {
      const unsigned mu = (unsigned)m;            // M < 2^31 checked by the launcher
      const unsigned t1 = mu / (unsigned)p.Wo;
      const int wo = (int)(mu - t1 * (unsigned)p.Wo);
      const int n = (int)(t1 / (unsigned)p.Ho);
      const int ho = (int)(t1 - (unsigned)n * (unsigned)p.Ho);
      float gy[8];
      if constexpr (KS == 3) {
        // loads are issued one filter row (3 taps) ahead of their use: 80 accumulators leave no room for all 9 vectors
        Vec16<__nv_bfloat16> gv = ld16(dy + m * p.C + cg * 8);
#pragma unroll
        for (int j = 0; j < 8; ++j) { gy[j] = __bfloat162float(gv.v[j]); acc[KK][j] += gy[j]; }
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
              for (int j = 0; j < 8; ++j) acc[r * 3 + s][j] = fmaf(gy[j], __bfloat162float(xv3[s].v[j]), acc[r * 3 + s][j]);
            }
          }
        }
        continue;
      }
      load8(dy + m * p.C + cg * 8, gy);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[KK][j] += gy[j];
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
          for (int j = 0; j < 8; ++j) acc[r * KS + s][j] = fmaf(gy[j], xv[j], acc[r * KS + s][j]);
        }
      }
    }
  }
#pragma unroll
  for (int k = 0; k <= KK; ++k) {
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) red[threadIdx.x * 8 + j] = acc[k][j];
    __syncthreads();
    fold_row_lanes<double, 1>(g, red, [&](int c, const double (&a)[1]) {
      part[((size_t)blockIdx.x * p.C + c) * (KK + 1) + k] = a[0];
    });
  }
}

// 3x3 weight gradient, stride 1 / 2: a thread owns ONE filter row r and FOUR consecutive output pixels of a row. It loads the 4
// dy vectors and the 3*S + 3 input vectors of input row oh*S + r - pad (all in flight before the first use) and keeps 3 taps x 8
// channels (+ the bias column on r == 0) of accumulators: 32 instead of 80, so two blocks per SM fit without serialising the
// loads filter row by filter row, and 7.5 / 11.25 vector loads per output pixel instead of 10. ty = lane * 3 + r: the block
// walks rows_t / 3 quads per step.
template <int kStride>
__global__ void __launch_bounds__(kThreads, 2) dw3x3_wgrad_quad_kernel(const __nv_bfloat16* __restrict__ x,
                                                                    const __nv_bfloat16* __restrict__ dy, double* part,
                                                                    DwParams p, const __grid_constant__ SlabGeo g) {
  __shared__ float red[kThreads * 8];
  const int tx = threadIdx.x % g.cg_t, ty = threadIdx.x / g.cg_t;
  const int r = ty % 3, lane = ty / 3, lanes = g.rows_t / 3;
  const int cg = blockIdx.y * g.cg_t + tx;
  const bool active = lane < lanes && cg < g.cg_total;
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
      for (int o = 0; o < 4; ++o) gv[o] = ld16_or_zero(dyp + (size_t)o * C, ow0 + o < p.Wo);
      if (hok) {
        const __nv_bfloat16* row = x + (((size_t)n * p.H + ih) * p.W) * C + cg * 8;
        const int iw0 = ow0 * kStride - p.pad;
#pragma unroll
        for (int c = 0; c < kIn; ++c) {
          const int iw = iw0 + c;
          xv[c] = ld16_or_zero(row + (size_t)iw * C, iw >= 0 && iw < p.W);
        }
      }
      float gy[4][8];
#pragma unroll
      for (int o = 0; o < 4; ++o)
#pragma unroll
        for (int j = 0; j < 8; ++j) gy[o][j] = __bfloat162float(gv[o].v[j]);
      if (r == 0) {
#pragma unroll
        for (int o = 0; o < 4; ++o)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[3][j] += gy[o][j];
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
              for (int j = 0; j < 8; ++j) acc[s2][j] = fmaf(gy[o][j], f[j], acc[s2][j]);
            }
          }
        }
      }
    }
  }
  const int nch = g.cg_t * 8;
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
      const int gcg = blockIdx.y * g.cg_t + ctx;
      if (gcg >= g.cg_total) continue;
      double a = 0.0;
      for (int l = 0; l < lanes; ++l) a += (double)red[(((l * 3 + rr) * g.cg_t) + ctx) * 8 + j];
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

// row blocks per SM of the weight-gradient kernels; hb_dwconv_wgrad_scratch_doubles sizes their partial sums for it
constexpr int kWgradPerSm = 2;

// HB_DISABLE_DW_QUAD set: the 3x3 launchers take the one-output kernels (dw3x3_kernel, dw_bwd_weight_kernel<3>) where they
// would take the four-output ones. Read once per process.
inline bool quad_kernels_on() {
  static const bool on = getenv("HB_DISABLE_DW_QUAD") == nullptr;
  return on;
}

// dw3x3_kernel with the stride as a template argument when it is 1 or 2
template <bool kBackward>
void launch_dw3x3(dim3 grid, cudaStream_t st, const __nv_bfloat16* src, const float* w, const float* bias,
                  __nv_bfloat16* dst, const DwParams& p, const SlabGeo& g) {
  const auto kernel = p.stride == 1 ? dw3x3_kernel<kBackward, 1> : p.stride == 2 ? dw3x3_kernel<kBackward, 2>
                                                                                  : dw3x3_kernel<kBackward, 0>;
  kernel<<<grid, kThreads, 0, st>>>(src, w, bias, dst, p, g);
}

// 0 when the geometry is supported (fills p), otherwise cudaErrorInvalidValue, before any launch or device query:
// N, C >= 1, C % 8 == 0 and a K x K filter window_out accepts on both axes.
int make_params(DwParams& p, int N, int H, int W, int C, int K, int stride, int pad) {
  int Ho, Wo;
  if (N < 1 || C < 1 || C % 8 != 0 || !window_out(H, K, stride, pad, 1, Ho) || !window_out(W, K, stride, pad, 1, Wo))
    return (int)cudaErrorInvalidValue;
  p = DwParams{N, H, W, C, Ho, Wo, K, stride, pad};
  return 0;
}

}  // namespace

extern "C" {

// y[N,Ho,Wo,C] = dwconv(x[N,H,W,C], w fp32 [C,K,K]) + bias; C % 8 == 0
int hb_dwconv_fwd_bf16(const void* x, const float* w, const float* bias, void* y, int N, int H, int W, int C, int K,
                       int stride, int pad, void* stream) {
  DwParams p;
  if (int rc = make_params(p, N, H, W, C, K, stride, pad)) return rc;
  const __nv_bfloat16* xb = (const __nv_bfloat16*)x;
  __nv_bfloat16* yb = (__nv_bfloat16*)y;
  cudaStream_t st = (cudaStream_t)stream;
  const long long M = (long long)N * p.Ho * p.Wo;
  if (K == 3 && M < 0x7fffffffLL) {
    const SlabGeo g = SlabGeo::make(C);
    if (quad_kernels_on() && (stride == 1 || stride == 2) && p.Wo >= 4) {
      const long long quads = (long long)N * p.Ho * ((p.Wo + 3) / 4);
      const auto kernel = stride == 1 ? dw3x3_quad_kernel<1, false> : dw3x3_quad_kernel<2, false>;
      kernel<<<g.grid(quads, 2, 2), kThreads, 0, st>>>(xb, w, bias, yb, N, H, W, p.Ho, p.Wo, C, pad, g);
    } else {
      launch_dw3x3<false>(g.grid(M, 3, 4), st, xb, w, bias, yb, p, g);
    }
  } else {
    dw_fwd_kernel<<<stream_grid((size_t)(M * (C / 8)), kThreads, 16), kThreads, 0, st>>>(xb, w, bias, yb, p);
  }
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_dwconv_bwd_data_bf16(const void* dy, const float* w, void* dx, int N, int H, int W, int C, int K, int stride,
                            int pad, void* stream) {
  DwParams p;
  if (int rc = make_params(p, N, H, W, C, K, stride, pad)) return rc;
  const __nv_bfloat16* dyb = (const __nv_bfloat16*)dy;
  __nv_bfloat16* dxb = (__nv_bfloat16*)dx;
  cudaStream_t st = (cudaStream_t)stream;
  const long long M = (long long)N * H * W;
  if (K == 3 && M < 0x7fffffffLL) {
    const SlabGeo g = SlabGeo::make(C);
    const long long quads = (long long)N * H * ((W + 3) / 4);
    if (quad_kernels_on() && stride == 1 && W >= 4 && pad <= 2) {
      // stride 1: the data gradient is the correlation of dy [N,Ho,Wo,C] with the flipped filter, padding 2 - pad
      dw3x3_quad_kernel<1, true><<<g.grid(quads, 2, 2), kThreads, 0, st>>>(dyb, w, nullptr, dxb, N, p.Ho, p.Wo, H, W, C,
                                                                           2 - pad, g);
    } else if (quad_kernels_on() && stride == 2 && pad == 1 && W >= 4) {
      dw3x3_dgrad_s2_quad_kernel<<<g.grid(quads, 2, 2), kThreads, 0, st>>>(dyb, w, dxb, N, H, W, p.Ho, p.Wo, C, g);
    } else {
      launch_dw3x3<true>(g.grid(M, 3, 4), st, dyb, w, nullptr, dxb, p, g);
    }
  } else {
    dw_bwd_data_kernel<<<stream_grid((size_t)(M * (C / 8)), kThreads, 16), kThreads, 0, st>>>(dyb, w, dxb, p);
  }
  HB_LAUNCH_CHECK();
  return 0;
}

// doubles of scratch hb_dwconv_bwd_weight_bf16 needs for C channels and a K x K filter (per-block partial sums); 0 for
// the shapes it refuses (K outside {1, 3, 5, 7})
size_t hb_dwconv_wgrad_scratch_doubles(int C, int K) {
  if (C <= 0 || C % 8 != 0 || (K != 1 && K != 3 && K != 5 && K != 7)) return 0;
  return (size_t)SlabGeo::make(C).max_blocks(kWgradPerSm) * C * (K * K + 1);
}

// dw fp32 [C,K,K], db fp32 [C] (or NULL); scratch: double[hb_dwconv_wgrad_scratch_doubles(C, K)]. K in {1, 3, 5, 7}.
int hb_dwconv_bwd_weight_bf16(const void* x, const void* dy, float* dw, float* db, double* scratch, int N, int H, int W,
                              int C, int K, int stride, int pad, void* stream) {
  DwParams p;
  if (int rc = make_params(p, N, H, W, C, K, stride, pad)) return rc;
  if (K != 1 && K != 3 && K != 5 && K != 7) return (int)cudaErrorInvalidValue;
  const long long M = (long long)N * p.Ho * p.Wo;
  if (M >= 0x7fffffffLL) return (int)cudaErrorInvalidValue;
  const __nv_bfloat16* xb = (const __nv_bfloat16*)x;
  const __nv_bfloat16* dyb = (const __nv_bfloat16*)dy;
  cudaStream_t st = (cudaStream_t)stream;
  const int KK = K * K;
  const SlabGeo g = SlabGeo::make(C);
  dim3 grid;
  if (quad_kernels_on() && K == 3 && (stride == 1 || stride == 2) && g.rows_t >= 3) {
    const long long quads = (long long)N * p.Ho * ((p.Wo + 3) / 4);
    grid = g.grid(quads, kWgradPerSm, 2, g.rows_t / 3);   // one quad per three row lanes
    const auto kernel = stride == 1 ? dw3x3_wgrad_quad_kernel<1> : dw3x3_wgrad_quad_kernel<2>;
    kernel<<<grid, kThreads, 0, st>>>(xb, dyb, scratch, p, g);
  } else {
    grid = g.grid(M, kWgradPerSm, 8);
    const auto kernel = K == 1 ? dw_bwd_weight_kernel<1> : K == 3 ? dw_bwd_weight_kernel<3>
                      : K == 5 ? dw_bwd_weight_kernel<5> : dw_bwd_weight_kernel<7>;
    kernel<<<grid, kThreads, 0, st>>>(xb, dyb, scratch, p, g);
  }
  HB_LAUNCH_CHECK();
  dw_weight_finalize_kernel<<<(C * (KK + 1) + 7) / 8, dim3(8, 32), 0, st>>>(scratch, (int)grid.x, dw, db, C, KK);
  HB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
