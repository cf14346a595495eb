// Lambda layer (reference holocron/nn/modules/lambda_layer.py:15-108, LambdaNetworks) over NHWC bf16 tensors, fp32
// accumulation. With dim_k = dk, dim_u = u, dim_v = dv, heads h and HW positions per sample:
//   sigma[b,u,k,m] = softmax_m(kproj[b,m,k*u+u])                                 (key softmax over the positions)
//   lc[b,k,v]      = sum_{u,m} sigma[b,u,k,m] * v[b,m,v*u+u]                       (content lambda)
//   lp[b,k,v,n]    = sum_{u,tap} R[k,u,tap] * v[b,n+tap,v*u+u]  (local, zero padded)  or
//                    sum_{m,u} pos_emb[n,m,k,u] * v[b,m,v*u+u]  (global: a GEMM, computed outside these kernels)
//   y[b,n,h*dv+v]  = sum_k q[b,n,h*dk+k] * (lc[b,k,v] + lp[b,k,v,n])
// The reference builds lp (B*dk*dv*HW fp32) with a conv3d and keeps it for autograd; the local kernels here never write it.
// The output and dq kernels form Qr = sum_k q * R per tap on the fly from a shared-memory halo of v (see DESIGN.md §3).
// Every reduction runs in a fixed order (no atomics) and nothing synchronises with the host.
//
// Layouts: q [B,HW,Cqp] (channel h*dk+k), k [B,HW,Ckp] (k*u+u), v [B,HW,Cvp] (v*u+u), y / dy [B,HW,Cop] (h*dv+v), all bf16
// with padding channels up to the pitch. Outputs get zeros there. The padding of q, k and dy is never read; that of v
// is (the halo kernels stage whole vectors and weight its lanes by zero) and must hold zeros; stats [B,dk*u,2] fp32 (row max, sum of exponentials); lc / dlc [B,dk,dv] fp32;
// Rt [r*r,u,dk] fp32 (R transposed tap-major); lp [B,HW,dk,dv] fp32 (global); dlp [B,HW,dk,dvp] bf16, dvp = dv rounded
// up to 8 (the transient per-position gradient of lp, sum_h q * dy); dvpos [B,HW,dv*u] fp32 (global share of dv).
#include <math.h>

#include <type_traits>

#include "nhwc.cuh"

namespace {

using namespace hb;
using bf16 = __nv_bfloat16;

constexpr int kThreads = 256;   // row kernels (content, backward content, dR)
constexpr int kTile = 8;        // output tile of the halo kernels: 8 x 8 positions, one thread per position and head
constexpr int kMaxR = 23;

struct LamParams {
  int B, H, W, HW, dk, u, heads, dv, r, Cqp, Ckp, Cvp, Cop, dvp;
};

__device__ __forceinline__ float bf(bf16 x) { return __bfloat162float(x); }

// (max, sum of exp(x - max)) pairs: combine b into a
__device__ __forceinline__ void lse_combine(float& ma, float& sa, float mb, float sb) {
  if (mb == -INFINITY) return;
  if (ma == -INFINITY) { ma = mb; sa = sb; return; }
  const float m = fmaxf(ma, mb);
  sa = sa * expf(ma - m) + sb * expf(mb - m);
  ma = m;
}

// Key softmax statistics and content lambda: one CTA per (k, b). For each of the u rows k*u+u' an online max / sum over
// the positions (fixed-order tree), then lc[b,k,:] = sum_m sum_u sigma * v, m-chunks of 256 with sigma staged in shared
// memory, lane = v (4 per lane), warp = m (stride 8), warps added in order.
__global__ void __launch_bounds__(kThreads) lam_content_kernel(const bf16* __restrict__ kt, const bf16* __restrict__ v,
                                                               float* __restrict__ stats, float* __restrict__ lc,
                                                               LamParams p) {
  __shared__ float sig[4][kThreads];
  __shared__ float red[kThreads / 32][128];
  __shared__ float mxs[kThreads], sms[kThreads];
  __shared__ float rowmax[4], rowsum[4];
  const int kk = blockIdx.x, b = blockIdx.y, t = threadIdx.x;
  const bf16* kb = kt + (size_t)b * p.HW * p.Ckp;
  const bf16* vb = v + (size_t)b * p.HW * p.Cvp;
  for (int uu = 0; uu < p.u; ++uu) {
    const int ch = kk * p.u + uu;
    float mx = -INFINITY, s = 0.f;
    for (int m = t; m < p.HW; m += kThreads) {
      const float x = bf(kb[(size_t)m * p.Ckp + ch]);
      // a -inf key has weight 0, as in torch.softmax; while mx is still -inf it would add exp(-inf - -inf) = NaN. A
      // row of -inf keys keeps (-inf, 0), so its sigma is NaN, as torch gives it.
      if (x == -INFINITY) continue;
      if (x > mx) { s = s * expf(mx - x) + 1.f; mx = x; }
      else s += expf(x - mx);
    }
    mxs[t] = mx;
    sms[t] = s;
    __syncthreads();
    for (int off = kThreads / 2; off > 0; off >>= 1) {
      if (t < off) lse_combine(mxs[t], sms[t], mxs[t + off], sms[t + off]);
      __syncthreads();
    }
    if (t == 0) {
      rowmax[uu] = mxs[0];
      rowsum[uu] = sms[0];
      float* st = stats + ((size_t)b * p.dk * p.u + ch) * 2;
      st[0] = mxs[0];
      st[1] = sms[0];
    }
    __syncthreads();
  }
  const int lane = t & 31, warp = t >> 5;
  for (int v0 = 0; v0 < p.dv; v0 += 128) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int m0 = 0; m0 < p.HW; m0 += kThreads) {
      const int cnt = min(kThreads, p.HW - m0);
      __syncthreads();
      if (t < cnt)
        for (int uu = 0; uu < p.u; ++uu)
          sig[uu][t] = __fdividef(expf(bf(kb[(size_t)(m0 + t) * p.Ckp + kk * p.u + uu]) - rowmax[uu]), rowsum[uu]);
      __syncthreads();
      for (int mm = warp; mm < cnt; mm += kThreads / 32) {
        const bf16* vr = vb + (size_t)(m0 + mm) * p.Cvp;
        for (int uu = 0; uu < p.u; ++uu) {
          const float sg = sig[uu][mm];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int vi = v0 + lane + 32 * i;
            if (vi < p.dv) acc[i] = fmaf(sg, bf(vr[vi * p.u + uu]), acc[i]);
          }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) red[warp][lane + 32 * i] = acc[i];
    __syncthreads();
    if (t < 128 && v0 + t < p.dv) {
      float s = 0.f;
      for (int w = 0; w < kThreads / 32; ++w) s += red[w][t];
      lc[((size_t)b * p.dk + kk) * p.dv + v0 + t] = s;
    }
    __syncthreads();
  }
}

// Copies the halo box [(kTile + r - 1)^2 pixels][U vectors] of v channels [v0*U, v0*U + 8U) around an output tile into
// shared memory.
template <int U>
__device__ __forceinline__ void stage_v(uint4* vs, const bf16* __restrict__ v, const LamParams& p, int b, int ty0, int tx0,
                                        int v0) {
  const int pad = p.r / 2, box = kTile + p.r - 1;
  stage_box(vs, v, (size_t)b * p.HW, p.H, p.W, p.Cvp, ty0 - pad, tx0 - pad, box, box, U, v0 * U / 8);
}

// Output: a CTA covers an 8 x 8 tile of one sample, thread = (position, head), dv in chunks of 8. Content term from lc,
// position term (local) from the v halo: per tap and u', qr = sum_k q[k] * Rt[tap,u',k], then acc[j] += qr * v[tap, j*U+u'].
// Global: lp read per position.
template <int DK, int U, bool kLocal>
__global__ void __launch_bounds__(512, 1) lam_out_kernel(const bf16* __restrict__ q, const bf16* __restrict__ v,
                                                      const float* __restrict__ Rt, const float* __restrict__ lc,
                                                      const float* __restrict__ lp, bf16* __restrict__ y, LamParams p,
                                                      int tiles_w) {
  extern __shared__ uint4 vs[];
  const int b = blockIdx.y;
  const int ty0 = (blockIdx.x / tiles_w) * kTile, tx0 = (blockIdx.x % tiles_w) * kTile;
  const int pos = threadIdx.x % (kTile * kTile), h = threadIdx.x / (kTile * kTile);
  const int py = pos / kTile, px = pos % kTile;
  const bool live = ty0 + py < p.H && tx0 + px < p.W;
  const size_t n = (size_t)b * p.HW + (live ? (ty0 + py) * p.W + tx0 + px : 0);
  const bf16* qp = q + n * p.Cqp + h * DK;
  float qr[kLocal ? DK : 1];
  if constexpr (kLocal) {
#pragma unroll
    for (int k = 0; k < DK; ++k) qr[k] = bf(qp[k]);
  }
  const float* lcb = lc + (size_t)b * DK * p.dv;
  const int box = kTile + p.r - 1, rr = p.r * p.r;
  const bool vec_out = p.dv % 8 == 0;
  bf16* yp = y + n * p.Cop + h * p.dv;
  for (int v0 = 0; v0 < p.dv; v0 += 8) {
    const int nv = min(8, p.dv - v0);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    if constexpr (kLocal) {
#pragma unroll
      for (int k = 0; k < DK; ++k)
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (j < nv) acc[j] = fmaf(qr[k], lcb[k * p.dv + v0 + j], acc[j]);
      __syncthreads();   // the previous chunk's taps are read
      stage_v<U>(vs, v, p, b, ty0, tx0, v0);
      if (live) {
        for (int t = 0; t < rr; ++t) {
          const int i = t / p.r, jj = t - i * p.r;
          const uint4* sp = vs + ((py + i) * box + px + jj) * U;
          Vec16<bf16> sv[U];
#pragma unroll
          for (int uv = 0; uv < U; ++uv) sv[uv].raw = sp[uv];
          const float* rt = Rt + (size_t)t * U * DK;
#pragma unroll
          for (int uu = 0; uu < U; ++uu) {
            float a = 0.f;
#pragma unroll
            for (int k = 0; k < DK; ++k) a = fmaf(qr[k], rt[uu * DK + k], a);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = fmaf(a, bf(sv[(j * U + uu) / 8].v[(j * U + uu) % 8]), acc[j]);
          }
        }
      }
    } else {
      const float* lpp = lp + n * DK * p.dv + v0;
#pragma unroll 1
      for (int k = 0; k < DK; ++k) {
        const float qk = bf(qp[k]);
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (j < nv) acc[j] = fmaf(qk, lcb[k * p.dv + v0 + j] + lpp[k * p.dv + j], acc[j]);
      }
    }
    if (live) {
      if (vec_out) {
        Vec16<bf16> o;
#pragma unroll
        for (int j = 0; j < 8; ++j) o.v[j] = __float2bfloat16_rn(acc[j]);
        st16(yp + v0, o);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (j < nv) yp[v0 + j] = __float2bfloat16_rn(acc[j]);
      }
    }
  }
  if (live && h == p.heads - 1)
    for (int c = p.heads * p.dv; c < p.Cop; ++c) y[n * p.Cop + c] = __float2bfloat16_rn(0.f);
}

// Backward, per-sample part, one CTA per (k, b): dlc[b,k,v] = sum_m sum_h q[m,h*dk+k] * dy[m,h*dv+v] (same layout of the
// reduction as the content kernel), then the softmax backward of each row k*u+u':
//   dsigma[m] = sum_v dlc[k,v] * v[m,v*u+u'],  dk[m] = sigma[m] * (dsigma[m] - sum_m' sigma * dsigma).
// The CTA with k = 0 also zeroes the padding channels of dk.
__global__ void __launch_bounds__(kThreads) lam_bwd_content_kernel(const bf16* __restrict__ q, const bf16* __restrict__ kt,
                                                                   const bf16* __restrict__ v, const bf16* __restrict__ dy,
                                                                   const float* __restrict__ stats,
                                                                   float* __restrict__ dlc, bf16* __restrict__ dkt,
                                                                   LamParams p) {
  extern __shared__ float dlc_s[];
  __shared__ float red[kThreads / 32][128];
  __shared__ float scratch[32];
  const int kk = blockIdx.x, b = blockIdx.y, t = threadIdx.x;
  const int lane = t & 31, warp = t >> 5;
  const size_t base = (size_t)b * p.HW;
  for (int v0 = 0; v0 < p.dv; v0 += 128) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int m = warp; m < p.HW; m += kThreads / 32) {
      const bf16* qm = q + (base + m) * p.Cqp + kk;
      const bf16* gm = dy + (base + m) * p.Cop;
      for (int h = 0; h < p.heads; ++h) {
        const float qv = bf(qm[h * p.dk]);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int vi = v0 + lane + 32 * i;
          if (vi < p.dv) acc[i] = fmaf(qv, bf(gm[h * p.dv + vi]), acc[i]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) red[warp][lane + 32 * i] = acc[i];
    __syncthreads();
    if (t < 128 && v0 + t < p.dv) {
      float s = 0.f;
      for (int w = 0; w < kThreads / 32; ++w) s += red[w][t];
      dlc[((size_t)b * p.dk + kk) * p.dv + v0 + t] = s;
      dlc_s[v0 + t] = s;
    }
    __syncthreads();
  }
  for (int uu = 0; uu < p.u; ++uu) {
    const int ch = kk * p.u + uu;
    const float* st = stats + ((size_t)b * p.dk * p.u + ch) * 2;
    const float mx = st[0], inv = __fdividef(1.f, st[1]);
    auto sig_dsig = [&](int m, float& sg, float& ds) {
      sg = expf(bf(kt[(base + m) * p.Ckp + ch]) - mx) * inv;
      const bf16* vm = v + (base + m) * p.Cvp + uu;
      float a = 0.f;
      for (int vi = 0; vi < p.dv; ++vi) a = fmaf(dlc_s[vi], bf(vm[vi * p.u]), a);
      ds = a;
    };
    float part = 0.f;
    for (int m = t; m < p.HW; m += kThreads) {
      float sg, ds;
      sig_dsig(m, sg, ds);
      part = fmaf(sg, ds, part);
    }
    const float tot = block_sum<float, true>(part, scratch);
    for (int m = t; m < p.HW; m += kThreads) {
      float sg, ds;
      sig_dsig(m, sg, ds);
      dkt[(base + m) * p.Ckp + ch] = __float2bfloat16_rn(sg * (ds - tot));
    }
  }
  if (kk == 0)
    for (int m = t; m < p.HW; m += kThreads)
      for (int c = p.dk * p.u; c < p.Ckp; ++c) dkt[(base + m) * p.Ckp + c] = __float2bfloat16_rn(0.f);
}

// dlp[b,n,k,v] = sum_h q[n,h*dk+k] * dy[n,h*dv+v] (bf16, v padded to dvp with zeros): a thread per 8 values.
__global__ void __launch_bounds__(kThreads) lam_dlp_kernel(const bf16* __restrict__ q, const bf16* __restrict__ dy,
                                                           bf16* __restrict__ dlp, LamParams p) {
  const int nvec = p.dvp / 8;
  const unsigned total = (unsigned)p.B * p.HW * p.dk * nvec;   // < 2^31, checked by make_params
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int vv = (int)(idx % (unsigned)nvec);
    const unsigned r = idx / (unsigned)nvec;
    const int k = (int)(r % (unsigned)p.dk);
    const size_t n = r / (unsigned)p.dk;
    const bf16* qn = q + n * p.Cqp + k;
    const bf16* gn = dy + n * p.Cop + vv * 8;
    float a[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = 0.f;
    for (int h = 0; h < p.heads; ++h) {
      const float qv = bf(qn[h * p.dk]);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (vv * 8 + j < p.dv) a[j] = fmaf(qv, bf(gn[h * p.dv + j]), a[j]);
    }
    Vec16<bf16> o;
#pragma unroll
    for (int j = 0; j < 8; ++j) o.v[j] = __float2bfloat16_rn(a[j]);
    st16(dlp + (size_t)idx * 8, o);
  }
}

// dq: same tiles and threads as the output kernel. dq[k] = sum_v dy[h,v] * (lc[k,v] + lp[k,v,n]); the local position part
// is sum_{tap,u'} Rt[tap,u',k] * d with d = sum_v dy[h,v] * v[n+tap, v*U+u'], from the same v halo.
template <int DK, int U, bool kLocal>
__global__ void __launch_bounds__(512, 1) lam_dq_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ v,
                                                     const float* __restrict__ Rt, const float* __restrict__ lc,
                                                     const float* __restrict__ lp, bf16* __restrict__ dq, LamParams p,
                                                     int tiles_w) {
  extern __shared__ uint4 vs[];
  const int b = blockIdx.y;
  const int ty0 = (blockIdx.x / tiles_w) * kTile, tx0 = (blockIdx.x % tiles_w) * kTile;
  const int pos = threadIdx.x % (kTile * kTile), h = threadIdx.x / (kTile * kTile);
  const int py = pos / kTile, px = pos % kTile;
  const bool live = ty0 + py < p.H && tx0 + px < p.W;
  const size_t n = (size_t)b * p.HW + (live ? (ty0 + py) * p.W + tx0 + px : 0);
  float acc[DK];
#pragma unroll
  for (int k = 0; k < DK; ++k) acc[k] = 0.f;
  const float* lcb = lc + (size_t)b * DK * p.dv;
  const int box = kTile + p.r - 1, rr = p.r * p.r;
  const bf16* gp = dy + n * p.Cop + h * p.dv;
  for (int v0 = 0; v0 < p.dv; v0 += 8) {
    const int nv = min(8, p.dv - v0);
    if constexpr (kLocal) {
      float g[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] = j < nv ? bf(gp[v0 + j]) : 0.f;
#pragma unroll
      for (int k = 0; k < DK; ++k) {
        float a = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (j < nv) a = fmaf(g[j], lcb[k * p.dv + v0 + j], a);
        acc[k] += a;
      }
      __syncthreads();
      stage_v<U>(vs, v, p, b, ty0, tx0, v0);
      if (live) {
        for (int t = 0; t < rr; ++t) {
          const int i = t / p.r, jj = t - i * p.r;
          const uint4* sp = vs + ((py + i) * box + px + jj) * U;
          Vec16<bf16> sv[U];
#pragma unroll
          for (int uv = 0; uv < U; ++uv) sv[uv].raw = sp[uv];
          const float* rt = Rt + (size_t)t * U * DK;
#pragma unroll
          for (int uu = 0; uu < U; ++uu) {
            float d = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) d = fmaf(g[j], bf(sv[(j * U + uu) / 8].v[(j * U + uu) % 8]), d);
#pragma unroll
            for (int k = 0; k < DK; ++k) acc[k] = fmaf(rt[uu * DK + k], d, acc[k]);
          }
        }
      }
    } else {
      const float* lpp = lp + n * DK * p.dv + v0;
#pragma unroll 1
      for (int j = 0; j < nv; ++j) {
        const float gj = bf(gp[v0 + j]);
#pragma unroll
        for (int k = 0; k < DK; ++k) acc[k] = fmaf(gj, lcb[k * p.dv + v0 + j] + lpp[k * p.dv + j], acc[k]);
      }
    }
  }
  if (!live) return;
  bf16* qo = dq + n * p.Cqp + h * DK;
#pragma unroll
  for (int k = 0; k < DK; ++k) qo[k] = __float2bfloat16_rn(acc[k]);
  if (h == p.heads - 1)
    for (int c = p.heads * DK; c < p.Cqp; ++c) dq[n * p.Cqp + c] = __float2bfloat16_rn(0.f);
}

// dv: a thread per (position m, 8 values of v) and every u'. Content path sum_k sigma[u',k,m] * dlc[k,v]; local position
// path sum_{k,tap} R[k,u',tap] * dlp[m - tap, k, v] (the correlation with the flipped R, taps read through L1);
// global: the GEMM share dvpos added. The last chunk also zeroes the padding channels.
template <int DK, int U, bool kLocal>
__global__ void lam_dv_kernel(const bf16* __restrict__ kt, const float* __restrict__ stats,
                                                          const float* __restrict__ dlc, const bf16* __restrict__ dlp,
                                                          const float* __restrict__ Rt, const float* __restrict__ dvpos,
                                                          bf16* __restrict__ dv, LamParams p) {
  const int nchunk = (p.dv + 7) / 8;
  const unsigned total = (unsigned)p.B * p.HW * nchunk;   // < 2^31, checked by make_params
  const int pad = p.r / 2;
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int ci = (int)(idx % (unsigned)nchunk);
    const unsigned nmu = idx / (unsigned)nchunk;
    const size_t nm = nmu;
    const int b = (int)(nmu / (unsigned)p.HW), m = (int)(nmu % (unsigned)p.HW);
    const int v0 = ci * 8, nv = min(8, p.dv - v0);
    float acc[U][8];
#pragma unroll
    for (int uu = 0; uu < U; ++uu)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[uu][j] = 0.f;
    const float* st = stats + (size_t)b * DK * U * 2;
    const bf16* km = kt + nm * p.Ckp;
    const float* dlb = dlc + (size_t)b * DK * p.dv + v0;
#pragma unroll
    for (int k = 0; k < DK; ++k)
#pragma unroll
      for (int uu = 0; uu < U; ++uu) {
        const int ch = k * U + uu;
        const float sg = __fdividef(expf(bf(km[ch]) - st[2 * ch]), st[2 * ch + 1]);
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (j < nv) acc[uu][j] = fmaf(sg, dlb[k * p.dv + j], acc[uu][j]);
      }
    if constexpr (kLocal) {
      const int y = m / p.W, x = m % p.W;
      for (int i = 0; i < p.r; ++i) {
        const int sy = y - i + pad;
        if (sy < 0 || sy >= p.H) continue;
        for (int jj = 0; jj < p.r; ++jj) {
          const int sx = x - jj + pad;
          if (sx < 0 || sx >= p.W) continue;
          const bf16* src = dlp + (((size_t)b * p.HW + sy * p.W + sx) * DK) * p.dvp + v0;
          const float* rt = Rt + (size_t)(i * p.r + jj) * U * DK;
#pragma unroll 4
          for (int k = 0; k < DK; ++k) {
            const Vec16<bf16> gv = ld16(src + (size_t)k * p.dvp);
#pragma unroll
            for (int uu = 0; uu < U; ++uu) {
              const float rw = rt[uu * DK + k];
#pragma unroll
              for (int j = 0; j < 8; ++j) acc[uu][j] = fmaf(rw, bf(gv.v[j]), acc[uu][j]);
            }
          }
        }
      }
    } else {
      const float* dp = dvpos + nm * p.dv * U + v0 * U;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (j < nv)
#pragma unroll
          for (int uu = 0; uu < U; ++uu) acc[uu][j] += dp[j * U + uu];
    }
    bf16* o = dv + nm * p.Cvp + v0 * U;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (j < nv)
#pragma unroll
        for (int uu = 0; uu < U; ++uu) o[j * U + uu] = __float2bfloat16_rn(acc[uu][j]);
    if (ci == nchunk - 1)
      for (int c = p.dv * U; c < p.Cvp; ++c) dv[nm * p.Cvp + c] = __float2bfloat16_rn(0.f);
  }
}

// dR partials, one CTA per (tap row i, sample b): part[b,k,u',i*r+j] = sum_n sum_v dlp[b,n,k,v] * v[b,n+tap,v*u+u'].
// The CTA walks the sample's 8 x 8 position tiles and 8-wide dim_v chunks; each step stages the tile's dlp [64][8][dk]
// and the strip of v its 8 rows read through tap row i (8 rows x (8 + r - 1) columns x 8u channels) in shared memory as
// fp32. A thread owns a 4 k x 4 j microtile of one u' (m = (k/4, u', j/4)) and one slice s of the 64 positions
// (s, s + S, ...): per position and v it loads 4 dlp values (one float4) and 4 v values for 16 FMAs. The S slices are
// added in order at the end. Everything runs in a fixed order.
constexpr int kDrTile = 8;
constexpr int kDrV = 8;

__host__ __device__ inline int dr_strip_w(int r) { return kDrTile + r + 2; }   // columns read by the last microtile

__global__ void __launch_bounds__(kThreads) lam_dr_partial_kernel(const bf16* __restrict__ dlp, const bf16* __restrict__ v,
                                                                  float* __restrict__ part, LamParams p) {
  extern __shared__ float dsm[];
  const int i = blockIdx.x, b = blockIdx.y, t = threadIdx.x;
  const int pad = p.r / 2, rr = p.r * p.r, u = p.u, dk = p.dk;
  const int sw = dr_strip_w(p.r), sc = kDrV * u;               // strip width, channels per strip pixel
  float* dls = dsm;                                             // [64 pos][kDrV][dk]
  float* vsm = dls + kDrTile * kDrTile * kDrV * dk;             // [kDrTile rows][sw][sc]
  const int jg = (p.r + 3) / 4, mt = (dk / 4) * u * jg;         // microtiles
  const int slices = kThreads / mt;
  const int m = t % mt, sl = t / mt;
  const int j0 = (m % jg) * 4, uu = (m / jg) % u, k0 = (m / jg / u) * 4;
  float acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[a][c] = 0.f;
  const int tiles_w = (p.W + kDrTile - 1) / kDrTile, tiles = tiles_w * ((p.H + kDrTile - 1) / kDrTile);
  const int cv = p.Cvp / 8;
  for (int tile = 0; tile < tiles; ++tile) {
    const int ty0 = (tile / tiles_w) * kDrTile, tx0 = (tile % tiles_w) * kDrTile;
    for (int v0 = 0; v0 < p.dvp; v0 += kDrV) {
      __syncthreads();   // the previous step's reads are done
      for (int e = t; e < kDrTile * kDrTile * dk; e += kThreads) {
        const int pos = e / dk, k = e - pos * dk;
        const int y = ty0 + pos / kDrTile, x = tx0 + pos % kDrTile;
        Vec16<bf16> g;
        if (y < p.H && x < p.W) g = ld16(dlp + (((size_t)b * p.HW + y * p.W + x) * dk + k) * p.dvp + v0);
        else g.raw = make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int vv = 0; vv < kDrV; ++vv) dls[(pos * kDrV + vv) * dk + k] = bf(g.v[vv]);
      }
      const int vec0 = v0 * u / 8;
      for (int e = t; e < kDrTile * sw * u; e += kThreads) {
        const int uv = e % u, pix = e / u;
        const int py = pix / sw, c = pix - py * sw;
        const int gy = ty0 + py + i - pad, gx = tx0 - pad + c;
        Vec16<bf16> g;
        if (c < kDrTile + p.r - 1 && gy >= 0 && gy < p.H && gx >= 0 && gx < p.W && vec0 + uv < cv)
          g = ld16(v + ((size_t)b * p.HW + gy * p.W + gx) * p.Cvp + (size_t)(vec0 + uv) * 8);
        else g.raw = make_uint4(0, 0, 0, 0);
        float* dst = vsm + (size_t)pix * sc + uv * 8;
#pragma unroll
        for (int q = 0; q < 8; ++q) dst[q] = bf(g.v[q]);
      }
      __syncthreads();
      if (sl < slices) {
        for (int pos = sl; pos < kDrTile * kDrTile; pos += slices) {
          const int py = pos / kDrTile, px = pos % kDrTile;
          const float* vrow = vsm + (size_t)(py * sw + px + j0) * sc + uu;
#pragma unroll
          for (int vv = 0; vv < kDrV; ++vv) {
            const float4 d4 = *reinterpret_cast<const float4*>(dls + (pos * kDrV + vv) * dk + k0);
            const float dd[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              const float x = vrow[c * sc + vv * u];
#pragma unroll
              for (int a = 0; a < 4; ++a) acc[a][c] = fmaf(dd[a], x, acc[a][c]);
            }
          }
        }
      }
    }
  }
  // slices in order: slice 0 .. S-1 through shared memory (reuses the dlp stage)
  __syncthreads();
  float* red = dsm;   // [slices][mt][16]
  if (sl < slices)
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int c = 0; c < 4; ++c) red[((size_t)sl * mt + m) * 16 + a * 4 + c] = acc[a][c];
  __syncthreads();
  if (t < mt) {
    float* out = part + (size_t)b * dk * u * rr;
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        if (j0 + c >= p.r) continue;
        float s = 0.f;
        for (int q = 0; q < slices; ++q) s += red[((size_t)q * mt + t) * 16 + a * 4 + c];
        out[((size_t)(k0 + a) * u + uu) * rr + i * p.r + j0 + c] = s;
      }
  }
}

size_t dr_smem_bytes(const LamParams& p) {
  const size_t stage = (size_t)kDrTile * kDrTile * kDrV * p.dk + (size_t)kDrTile * dr_strip_w(p.r) * kDrV * p.u;
  const size_t red = (size_t)kThreads * 16;
  return (stage > red ? stage : red) * sizeof(float);
}

// dR[k,u',tap] = sum_b part[b,k,u',tap], samples in order
__global__ void __launch_bounds__(kThreads) lam_dr_reduce_kernel(const float* __restrict__ part, float* __restrict__ dR,
                                                                 int B, int per_sample) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < per_sample; e += gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += part[(size_t)b * per_sample + e];
    dR[e] = s;
  }
}

// 0 when the shape is supported (fills p), otherwise cudaErrorInvalidValue
int make_params(LamParams& p, int B, int H, int W, int dk, int u, int heads, int dv, int r, int Cqp, int Ckp, int Cvp,
                int Cop) {
  if (B <= 0 || H <= 0 || W <= 0 || (dk != 8 && dk != 16 && dk != 32) || u < 1 || u > 4 || heads < 1 || heads > 8 ||
      dv < 1 || r < 0 || r > kMaxR || (r > 0 && r % 2 == 0) || Cqp < heads * dk || Ckp < dk * u || Cvp < dv * u ||
      Cop < heads * dv || Cqp % 8 || Ckp % 8 || Cvp % 8 || Cop % 8 || B > 65535)
    return (int)cudaErrorInvalidValue;
  p = LamParams{B, H, W, H * W, dk, u, heads, dv, r, Cqp, Ckp, Cvp, Cop, (dv + 7) / 8 * 8};
  // 32-bit element indices in the grid-stride kernels
  long long cmax = Cqp;
  for (int c : {Ckp, Cvp, Cop}) cmax = c > cmax ? c : cmax;
  if ((long long)B * H * W * cmax >= 0x7fffffffLL || (long long)B * H * W * dk * p.dvp >= 0x7fffffffLL)
    return (int)cudaErrorInvalidValue;
  return 0;
}

struct HaloGrid {
  dim3 grid, block;
  size_t smem;
  int tiles_w;
};

HaloGrid halo_grid(const LamParams& p, int U) {
  HaloGrid g;
  g.tiles_w = (p.W + kTile - 1) / kTile;
  g.grid = dim3((unsigned)(g.tiles_w * ((p.H + kTile - 1) / kTile)), (unsigned)p.B);
  g.block = dim3((unsigned)(kTile * kTile * p.heads));
  const int box = kTile + p.r - 1;
  g.smem = p.r > 0 ? (size_t)box * box * U * 16 : 0;
  return g;
}

template <int V> using Int = std::integral_constant<int, V>;

// f(Int<dk>{}) and f(Int<u>{}) for the dk and u make_params accepts
template <typename F> int with_dk(int dk, F&& f) {
  switch (dk) {
    case 8: return f(Int<8>{});
    case 16: return f(Int<16>{});
    default: return f(Int<32>{});
  }
}

template <typename F> int with_u(int u, F&& f) {
  switch (u) {
    case 1: return f(Int<1>{});
    case 2: return f(Int<2>{});
    case 3: return f(Int<3>{});
    default: return f(Int<4>{});
  }
}

// Dispatch of the (DK, U, local) instantiations; the global variant does not read v in these kernels and takes U = 1.
template <template <int, int, bool> class Launch, typename... Args>
int dispatch(const LamParams& p, Args... args) {
  return with_dk(p.dk, [&](auto dk) {
    constexpr int DK = decltype(dk)::value;
    if (p.r == 0) return Launch<DK, 1, false>::run(p, args...);
    return with_u(p.u, [&](auto u) { return Launch<DK, decltype(u)::value, true>::run(p, args...); });
  });
}

template <int DK, int U, bool kLocal>
struct OutLaunch {
  static int run(const LamParams& p, const bf16* q, const bf16* v, const float* Rt, const float* lc, const float* lp,
                 bf16* y, cudaStream_t st) {
    const HaloGrid g = halo_grid(p, U);
    if (cudaError_t e = allow_smem(lam_out_kernel<DK, U, kLocal>, g.smem, g.smem)) return (int)e;
    lam_out_kernel<DK, U, kLocal><<<g.grid, g.block, g.smem, st>>>(q, v, Rt, lc, lp, y, p, g.tiles_w);
    HB_LAUNCH_CHECK();
    return 0;
  }
};

template <int DK, int U, bool kLocal>
struct DqLaunch {
  static int run(const LamParams& p, const bf16* dy, const bf16* v, const float* Rt, const float* lc, const float* lp,
                 bf16* dq, cudaStream_t st) {
    const HaloGrid g = halo_grid(p, U);
    if (cudaError_t e = allow_smem(lam_dq_kernel<DK, U, kLocal>, g.smem, g.smem)) return (int)e;
    lam_dq_kernel<DK, U, kLocal><<<g.grid, g.block, g.smem, st>>>(dy, v, Rt, lc, lp, dq, p, g.tiles_w);
    HB_LAUNCH_CHECK();
    return 0;
  }
};

template <int DK, int U, bool kLocal>
struct DvLaunch {
  static int run(const LamParams& p, const bf16* kt, const float* stats, const float* dlc, const bf16* dlp,
                 const float* Rt, const float* dvpos, bf16* dv, cudaStream_t st) {
    const size_t total = (size_t)p.B * p.HW * ((p.dv + 7) / 8);
    lam_dv_kernel<DK, U, kLocal><<<stream_grid(total, kThreads, 16), kThreads, 0, st>>>(kt, stats, dlc, dlp, Rt, dvpos,
                                                                                        dv, p);
    HB_LAUNCH_CHECK();
    return 0;
  }
};

}  // namespace

extern "C" {

#define HB_LAM_GEOM int B, int H, int W, int dk, int u, int heads, int dv, int r, int Cqp, int Ckp, int Cvp, int Cop
#define HB_LAM_PARAMS                                                                    \
  LamParams p;                                                                           \
  if (int rc = make_params(p, B, H, W, dk, u, heads, dv, r, Cqp, Ckp, Cvp, Cop)) return rc; \
  cudaStream_t st = (cudaStream_t)stream;

int hb_lambda_content_fwd_bf16(const void* k, const void* v, float* stats, float* lc, HB_LAM_GEOM, void* stream) {
  HB_LAM_PARAMS
  lam_content_kernel<<<dim3((unsigned)dk, (unsigned)B), kThreads, 0, st>>>((const bf16*)k, (const bf16*)v, stats, lc, p);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_lambda_out_fwd_bf16(const void* q, const void* v, const float* Rt, const float* lc, const float* lp, void* y,
                           HB_LAM_GEOM, void* stream) {
  HB_LAM_PARAMS
  if (r > 0 ? !Rt : !lp) return (int)cudaErrorInvalidValue;
  return dispatch<OutLaunch>(p, (const bf16*)q, (const bf16*)v, Rt, lc, lp, (bf16*)y, st);
}

int hb_lambda_bwd_content_bf16(const void* q, const void* k, const void* v, const void* dy, const float* stats,
                               float* dlc, void* dk_out, HB_LAM_GEOM, void* stream) {
  HB_LAM_PARAMS
  lam_bwd_content_kernel<<<dim3((unsigned)dk, (unsigned)B), kThreads, (size_t)dv * sizeof(float), st>>>(
      (const bf16*)q, (const bf16*)k, (const bf16*)v, (const bf16*)dy, stats, dlc, (bf16*)dk_out, p);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_lambda_dlp_bf16(const void* q, const void* dy, void* dlp, HB_LAM_GEOM, void* stream) {
  HB_LAM_PARAMS
  const size_t total = (size_t)B * p.HW * dk * (p.dvp / 8);
  lam_dlp_kernel<<<stream_grid(total, kThreads, 16), kThreads, 0, st>>>((const bf16*)q, (const bf16*)dy, (bf16*)dlp, p);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_lambda_bwd_q_bf16(const void* dy, const void* v, const float* Rt, const float* lc, const float* lp, void* dq,
                         HB_LAM_GEOM, void* stream) {
  HB_LAM_PARAMS
  if (r > 0 ? !Rt : !lp) return (int)cudaErrorInvalidValue;
  return dispatch<DqLaunch>(p, (const bf16*)dy, (const bf16*)v, Rt, lc, lp, (bf16*)dq, st);
}

int hb_lambda_bwd_v_bf16(const void* k, const float* stats, const float* dlc, const void* dlp, const float* Rt,
                         const float* dvpos, void* dv_out, HB_LAM_GEOM, void* stream) {
  HB_LAM_PARAMS
  if (r > 0 ? (!Rt || !dlp) : !dvpos) return (int)cudaErrorInvalidValue;
  const bf16* kb = (const bf16*)k;
  const bf16* gb = (const bf16*)dlp;
  bf16* o = (bf16*)dv_out;
  // unlike the output and dq kernels, the global variant of dv runs with the layer's u
  return with_dk(dk, [&](auto d) {
    return with_u(u, [&](auto uu) {
      constexpr int DK = decltype(d)::value, U = decltype(uu)::value;
      return r > 0 ? DvLaunch<DK, U, true>::run(p, kb, stats, dlc, gb, Rt, dvpos, o, st)
                   : DvLaunch<DK, U, false>::run(p, kb, stats, dlc, gb, Rt, dvpos, o, st);
    });
  });
}

// scratch: B * dk * u * r * r floats (the per-sample partials)
int hb_lambda_bwd_r_bf16(const void* dlp, const void* v, float* scratch, float* dR, HB_LAM_GEOM, void* stream) {
  HB_LAM_PARAMS
  if (r == 0) return (int)cudaErrorInvalidValue;
  const size_t smem = dr_smem_bytes(p);
  if (cudaError_t e = allow_smem(lam_dr_partial_kernel, smem, smem)) return (int)e;
  lam_dr_partial_kernel<<<dim3((unsigned)r, (unsigned)B), kThreads, smem, st>>>((const bf16*)dlp, (const bf16*)v, scratch, p);
  HB_LAUNCH_CHECK();
  const int per = dk * u * r * r;
  lam_dr_reduce_kernel<<<(per + kThreads - 1) / kThreads, kThreads, 0, st>>>(scratch, dR, B, per);
  HB_LAUNCH_CHECK();
  return 0;
}

#undef HB_LAM_PARAMS
#undef HB_LAM_GEOM

}  // extern "C"
