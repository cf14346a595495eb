// Involution (reference holocron/nn/modules/conv.py:441-499) over NHWC bf16 tensors, fp32 accumulation:
//   y[n, o, c] = sum_t ker[n, o, g(c) * K^2 + t] * x[n, o * s - p + dil * (i_t, j_t), c],   g(c) = c / (C / G)
// x [N,H,W,Cp], ker [N,Ho,Wo,Kp] (the zero-padded span output), y [N,Ho,Wo,Cp]. The reference materialises the unfolded
// input (N*C*K^2*Ho*Wo elements) and a product of the same size; these kernels read x through a shared-memory halo tile
// and never build either.
//
// Every thread owns one pixel x 8 consecutive channels (one 128-bit vector). Channels c >= C (the zero padding up to Cp)
// are written as zeros; those of x and dy, and the columns G*K^2 .. Kp-1 of ker, are never read. "Uniform" vectors (C/G % 8 == 0, the RedNet case) have all 8 channels in one group, so a pixel's
// K^2 weights of that group are loaded once into registers; "mixed" vectors (e.g. C = 12, G = 6) look the group up per
// channel. Nothing here synchronises with the host; reductions run in a fixed order (no atomics).
#include <type_traits>

#include "nhwc.cuh"

namespace {

using namespace hb;
using bf16 = __nv_bfloat16;

constexpr int kThreads = 256;
constexpr int kTileW = 8;                    // output columns of a CTA tile; rows = kThreads / (nv * kTileW)
constexpr size_t kSmemMax = 112 * 1024;      // halo tile budget: two CTAs per SM

struct InvParams {
  int N, H, W, C, Cp, Ho, Wo, Kp, G, stride, pad, dil;
};

// Tile geometry shared by the host launchers and the kernels: nv channel vectors per pixel, th x kTileW output pixels,
// and the input box (halo included) those pixels read.
struct Tile {
  int nv, th, tiles_w, tiles_h, slabs, in_h, in_w;
  size_t smem;
  int threads() const { return nv * kTileW * th; }
};

Tile make_tile(const InvParams& p, int K, int nv) {
  Tile t;
  t.nv = nv;
  t.th = kThreads / (nv * kTileW);
  const int reach = p.dil * (K - 1) + 1;
  t.in_w = (kTileW - 1) * p.stride + reach;
  for (;;) {
    t.in_h = (t.th - 1) * p.stride + reach;
    t.smem = (size_t)t.in_h * t.in_w * nv * 16;
    if (t.smem <= kSmemMax || t.th == 1) break;
    t.th /= 2;
  }
  t.tiles_w = (p.Wo + kTileW - 1) / kTileW;
  t.tiles_h = (p.Ho + t.th - 1) / t.th;
  t.slabs = (p.Cp / 8 + nv - 1) / nv;
  return t;
}

// Forward. kSmem = false (only when a dilated halo box exceeds kSmemMax) reads the taps from global memory instead.
template <int K, bool kUniform, bool kSmem>
__global__ void __launch_bounds__(kThreads) inv_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ ker,
                                                           bf16* __restrict__ y, InvParams p, Tile tl) {
  extern __shared__ uint4 xs[];
  constexpr int KK = K * K;
  const int n = blockIdx.z;
  const int oy0 = (blockIdx.x / tl.tiles_w) * tl.th, ox0 = (blockIdx.x % tl.tiles_w) * kTileW;
  const int vbase = blockIdx.y * tl.nv;
  if (kSmem)
    stage_box(xs, x, (size_t)n * p.H * p.W, p.H, p.W, p.Cp, oy0 * p.stride - p.pad, ox0 * p.stride - p.pad, tl.in_h,
              tl.in_w, tl.nv, vbase);
  const int v = threadIdx.x % tl.nv, pix = threadIdx.x / tl.nv;
  const int ty = pix / kTileW, tx = pix % kTileW;
  const int oy = oy0 + ty, ox = ox0 + tx, cvec = vbase + v;
  if (oy >= p.Ho || ox >= p.Wo || cvec >= p.Cp / 8) return;
  const int c0 = cvec * 8, cg = p.C / p.G;
  const size_t o = ((size_t)n * p.Ho + oy) * p.Wo + ox;
  const bf16* kp = ker + o * p.Kp;
  auto tap = [&](int i, int j) {
    Vec16<bf16> xv;
    if (kSmem) {
      xv.raw = xs[((ty * p.stride + i * p.dil) * tl.in_w + tx * p.stride + j * p.dil) * tl.nv + v];
    } else {
      const int hi = oy * p.stride - p.pad + i * p.dil, wi = ox * p.stride - p.pad + j * p.dil;
      if (hi >= 0 && hi < p.H && wi >= 0 && wi < p.W) xv = ld16(x + (((size_t)n * p.H + hi) * p.W + wi) * p.Cp + c0);
      else xv.raw = make_uint4(0, 0, 0, 0);
    }
    return xv;
  };
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if constexpr (kUniform) {
    const bf16* kg = kp + (c0 / cg) * KK;
    float w[KK];
#pragma unroll
    for (int t = 0; t < KK; ++t) w[t] = __bfloat162float(kg[t]);
#pragma unroll
    for (int i = 0; i < K; ++i)
#pragma unroll
      for (int j = 0; j < K; ++j) {
        const Vec16<bf16> xv = tap(i, j);
#pragma unroll
        for (int l = 0; l < 8; ++l) acc[l] = fmaf(w[i * K + j], __bfloat162float(xv.v[l]), acc[l]);
      }
  } else {
    int goff[8];
    bool live[8];
#pragma unroll
    for (int l = 0; l < 8; ++l) {
      live[l] = c0 + l < p.C;
      goff[l] = live[l] ? ((c0 + l) / cg) * KK : 0;
    }
#pragma unroll
    for (int i = 0; i < K; ++i)
#pragma unroll
      for (int j = 0; j < K; ++j) {
        const Vec16<bf16> xv = tap(i, j);
#pragma unroll
        for (int l = 0; l < 8; ++l)
          if (live[l]) acc[l] = fmaf(__bfloat162float(kp[goff[l] + i * K + j]), __bfloat162float(xv.v[l]), acc[l]);
      }
  }
  store8(y + o * p.Cp + c0, acc);
}

// Data gradient, gather form: dx[n, h, w, c] = sum over the taps t whose source output pixel
// (h + p - dil * i_t, w + p - dil * j_t) / s exists (exact division) of ker[n, o, g(c) * K^2 + t] * dy[n, o, c].
// One thread per input pixel x 8 channels, every element written once.
template <int K, bool kUniform>
__global__ void __launch_bounds__(kThreads) inv_bwd_data_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ ker,
                                                                bf16* __restrict__ dx, InvParams p) {
  constexpr int KK = K * K;
  const unsigned cv = p.Cp / 8;
  const unsigned total = (unsigned)p.N * p.H * p.W * cv;   // < 2^31, checked by the launcher
  const int cg = p.C / p.G;
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const unsigned cvec = idx % cv;
    unsigned t = idx / cv;
    const int wi = (int)(t % (unsigned)p.W);
    t /= (unsigned)p.W;
    const int hi = (int)(t % (unsigned)p.H);
    const int n = (int)(t / (unsigned)p.H);
    const int c0 = (int)cvec * 8;
    int goff[8];
    bool live[8];
#pragma unroll
    for (int l = 0; l < 8; ++l) {
      live[l] = c0 + l < p.C;
      goff[l] = live[l] ? ((c0 + l) / cg) * KK : 0;
    }
    float acc[8];
#pragma unroll
    for (int l = 0; l < 8; ++l) acc[l] = 0.f;
#pragma unroll
    for (int i = 0; i < K; ++i) {
      const int hn = hi + p.pad - i * p.dil;
      if (hn < 0 || hn % p.stride != 0) continue;
      const int ho = hn / p.stride;
      if (ho >= p.Ho) continue;
#pragma unroll
      for (int j = 0; j < K; ++j) {
        const int wn = wi + p.pad - j * p.dil;
        if (wn < 0 || wn % p.stride != 0) continue;
        const int wo = wn / p.stride;
        if (wo >= p.Wo) continue;
        const size_t o = ((size_t)n * p.Ho + ho) * p.Wo + wo;
        const Vec16<bf16> g = ld16(dy + o * p.Cp + c0);
        const bf16* kp = ker + o * p.Kp + i * K + j;
        if constexpr (kUniform) {
          const float w = __bfloat162float(kp[goff[0]]);
#pragma unroll
          for (int l = 0; l < 8; ++l) acc[l] = fmaf(w, __bfloat162float(g.v[l]), acc[l]);
        } else {
#pragma unroll
          for (int l = 0; l < 8; ++l)
            if (live[l]) acc[l] = fmaf(__bfloat162float(kp[goff[l]]), __bfloat162float(g.v[l]), acc[l]);
        }
      }
    }
    store8(dx + (size_t)idx * 8, acc);
  }
}

// Kernel gradient for uniform vectors whose group spans vg = C/G/8 in {1, 2, 4, 8} vectors: each thread forms the K^2
// products dy . x(tap) over its 8 channels (fixed order), then the vg lanes of a group - adjacent lanes of one pixel -
// add theirs with an xor butterfly (every lane ends with the same bits), and lane r of the group writes the taps
// t = r (mod vg). The x taps come from the same shared-memory halo tile as the forward pass. The thread of the first
// vector of a pixel also writes the padding columns G*K^2 .. Kp-1 as zeros.
template <int K>
__global__ void __launch_bounds__(kThreads) inv_bwd_kernel_kernel(const bf16* __restrict__ x, const bf16* __restrict__ dy,
                                                                  bf16* __restrict__ dker, InvParams p, Tile tl, int vg) {
  extern __shared__ uint4 xs[];
  constexpr int KK = K * K;
  const int n = blockIdx.z;
  const int oy0 = (blockIdx.x / tl.tiles_w) * tl.th, ox0 = (blockIdx.x % tl.tiles_w) * kTileW;
  const int vbase = blockIdx.y * tl.nv;
  stage_box(xs, x, (size_t)n * p.H * p.W, p.H, p.W, p.Cp, oy0 * p.stride - p.pad, ox0 * p.stride - p.pad, tl.in_h,
            tl.in_w, tl.nv, vbase);
  const int v = threadIdx.x % tl.nv, pix = threadIdx.x / tl.nv;
  const int ty = pix / kTileW, tx = pix % kTileW;
  const int oy = oy0 + ty, ox = ox0 + tx, cvec = vbase + v;
  // a whole group is live or dead together (cv is a multiple of vg), so the butterfly never mixes the two; every lane
  // still runs it because the shuffles name the full warp
  const bool live = oy < p.Ho && ox < p.Wo && cvec < p.Cp / 8;
  const size_t o = ((size_t)n * p.Ho + (live ? oy : 0)) * p.Wo + (live ? ox : 0);
  float g[8];
  {
    Vec16<bf16> gv;
    if (live) gv = ld16(dy + o * p.Cp + cvec * 8);
    else gv.raw = make_uint4(0, 0, 0, 0);
#pragma unroll
    for (int l = 0; l < 8; ++l) g[l] = __bfloat162float(gv.v[l]);
  }
  float s[KK];
  const uint4* xb = xs + ((ty * p.stride) * tl.in_w + tx * p.stride) * tl.nv + v;
#pragma unroll
  for (int i = 0; i < K; ++i)
#pragma unroll
    for (int j = 0; j < K; ++j) {
      Vec16<bf16> xv;
      xv.raw = xb[(i * p.dil * tl.in_w + j * p.dil) * tl.nv];
      float a = 0.f;
#pragma unroll
      for (int l = 0; l < 8; ++l) a = fmaf(g[l], __bfloat162float(xv.v[l]), a);
      s[i * K + j] = a;
    }
  for (int off = 1; off < vg; off <<= 1) {
#pragma unroll
    for (int t = 0; t < KK; ++t) s[t] += __shfl_xor_sync(0xffffffffu, s[t], off);
  }
  if (!live) return;
  const int cg = p.C / p.G;
  bf16* kp = dker + o * p.Kp;
  bf16* kg = kp + (cvec * 8 / cg) * KK;
  const int r = cvec % vg;
#pragma unroll
  for (int t = 0; t < KK; ++t)
    if (t % vg == r) kg[t] = __float2bfloat16_rn(s[t]);
  if (cvec == 0)
    for (int k = p.G * KK; k < p.Kp; ++k) kp[k] = __float2bfloat16_rn(0.f);
}

// Kernel gradient for every other channel layout (mixed vectors, C/G not a power-of-two multiple of 8 up to 64, or a
// halo box larger than kSmemMax): one thread per element of dker [N,Ho,Wo,Kp], the group's channels summed in order.
__global__ void __launch_bounds__(kThreads) inv_bwd_kernel_generic_kernel(const bf16* __restrict__ x,
                                                                          const bf16* __restrict__ dy,
                                                                          bf16* __restrict__ dker, InvParams p, int K) {
  const int KK = K * K, cg = p.C / p.G;
  const unsigned total = (unsigned)p.N * p.Ho * p.Wo * p.Kp;   // < 2^31, checked by the launcher
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int k = (int)(idx % (unsigned)p.Kp);
    const unsigned o = idx / (unsigned)p.Kp;
    float a = 0.f;
    if (k < p.G * KK) {
      const int ox = (int)(o % (unsigned)p.Wo);
      const unsigned t = o / (unsigned)p.Wo;
      const int oy = (int)(t % (unsigned)p.Ho);
      const int n = (int)(t / (unsigned)p.Ho);
      const int gi = k / KK, tp = k % KK;
      const int hi = oy * p.stride - p.pad + (tp / K) * p.dil, wi = ox * p.stride - p.pad + (tp % K) * p.dil;
      if (hi >= 0 && hi < p.H && wi >= 0 && wi < p.W) {
        const bf16* dp = dy + (size_t)o * p.Cp + gi * cg;
        const bf16* xp = x + (((size_t)n * p.H + hi) * p.W + wi) * p.Cp + gi * cg;
        for (int c = 0; c < cg; ++c) a = fmaf(__bfloat162float(dp[c]), __bfloat162float(xp[c]), a);
      }
    }
    dker[idx] = __float2bfloat16_rn(a);
  }
}

// every 8-channel vector lies inside one group and no vector is padding
bool uniform_vectors(const InvParams& p) { return (p.C / p.G) % 8 == 0 && p.Cp == p.C; }

template <int K, bool kUniform>
int launch_fwd(const bf16* x, const bf16* ker, bf16* y, const InvParams& p, cudaStream_t st) {
  const int cv = p.Cp / 8;
  const Tile tl = make_tile(p, K, cv >= 4 ? 4 : (cv >= 2 ? 2 : 1));
  const dim3 grid((unsigned)(tl.tiles_w * tl.tiles_h), (unsigned)tl.slabs, (unsigned)p.N);
  if (tl.smem <= kSmemMax) {
    if (cudaError_t e = allow_smem(inv_fwd_kernel<K, kUniform, true>, tl.smem, kSmemMax)) return (int)e;
    inv_fwd_kernel<K, kUniform, true><<<grid, tl.threads(), tl.smem, st>>>(x, ker, y, p, tl);
  } else {
    inv_fwd_kernel<K, kUniform, false><<<grid, tl.threads(), 0, st>>>(x, ker, y, p, tl);
  }
  HB_LAUNCH_CHECK();
  return 0;
}

template <int K>
int launch_bwd_kernel(const bf16* x, const bf16* dy, bf16* dker, const InvParams& p, cudaStream_t st) {
  const int cv = p.Cp / 8;
  const int vg = uniform_vectors(p) ? p.C / p.G / 8 : 0;
  if (vg == 1 || vg == 2 || vg == 4 || vg == 8) {
    int nv = cv >= 4 ? 4 : (cv >= 2 ? 2 : 1);
    if (nv < vg) nv = vg;
    const Tile tl = make_tile(p, K, nv);
    if (tl.smem <= kSmemMax) {
      if (cudaError_t e = allow_smem(inv_bwd_kernel_kernel<K>, tl.smem, kSmemMax)) return (int)e;
      const dim3 grid((unsigned)(tl.tiles_w * tl.tiles_h), (unsigned)tl.slabs, (unsigned)p.N);
      inv_bwd_kernel_kernel<K><<<grid, tl.threads(), tl.smem, st>>>(x, dy, dker, p, tl, vg);
      HB_LAUNCH_CHECK();
      return 0;
    }
  }
  const size_t total = (size_t)p.N * p.Ho * p.Wo * p.Kp;
  inv_bwd_kernel_generic_kernel<<<stream_grid(total, kThreads, 16), kThreads, 0, st>>>(x, dy, dker, p, K);
  HB_LAUNCH_CHECK();
  return 0;
}

// 0 when the shape is supported (fills p), otherwise cudaErrorInvalidValue
int make_params(InvParams& p, int N, int H, int W, int C, int Cp, int Kp, int K, int G, int stride, int pad, int dil) {
  if (N <= 0 || C <= 0 || G <= 0 || C % G != 0 || Cp < C || Cp % 8 != 0 || Kp < G * K * K ||
      (K != 1 && K != 3 && K != 5 && K != 7))
    return (int)cudaErrorInvalidValue;
  int Ho, Wo;
  if (!window_out(H, K, stride, pad, dil, Ho) || !window_out(W, K, stride, pad, dil, Wo) || N > 65535)
    return (int)cudaErrorInvalidValue;
  p = InvParams{N, H, W, C, Cp, Ho, Wo, Kp, G, stride, pad, dil};
  // 32-bit element indices in the grid-stride kernels
  if ((long long)N * H * W * Cp >= 0x7fffffffLL || (long long)N * p.Ho * p.Wo * (Cp > Kp ? Cp : Kp) >= 0x7fffffffLL)
    return (int)cudaErrorInvalidValue;
  return 0;
}

// f(std::integral_constant<int, K>{}) for the K make_params accepts
template <typename F> int with_k(int K, F&& f) {
  switch (K) {
    case 1: return f(std::integral_constant<int, 1>{});
    case 3: return f(std::integral_constant<int, 3>{});
    case 5: return f(std::integral_constant<int, 5>{});
    default: return f(std::integral_constant<int, 7>{});
  }
}

}  // namespace

extern "C" {

int hb_involution_fwd_bf16(const void* x, const void* ker, void* y, int N, int H, int W, int C, int Cp, int Kp, int K,
                           int G, int stride, int pad, int dil, void* stream) {
  InvParams p;
  if (int rc = make_params(p, N, H, W, C, Cp, Kp, K, G, stride, pad, dil)) return rc;
  const bf16* xb = (const bf16*)x;
  const bf16* kb = (const bf16*)ker;
  bf16* yb = (bf16*)y;
  cudaStream_t st = (cudaStream_t)stream;
  const bool u = uniform_vectors(p);
  return with_k(K, [&](auto k) {
    constexpr int KK = decltype(k)::value;
    return u ? launch_fwd<KK, true>(xb, kb, yb, p, st) : launch_fwd<KK, false>(xb, kb, yb, p, st);
  });
}

int hb_involution_bwd_data_bf16(const void* dy, const void* ker, void* dx, int N, int H, int W, int C, int Cp, int Kp,
                                int K, int G, int stride, int pad, int dil, void* stream) {
  InvParams p;
  if (int rc = make_params(p, N, H, W, C, Cp, Kp, K, G, stride, pad, dil)) return rc;
  const bf16* dyb = (const bf16*)dy;
  const bf16* kb = (const bf16*)ker;
  bf16* dxb = (bf16*)dx;
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid(stream_grid((size_t)N * H * W * (Cp / 8), kThreads, 16));
  const bool u = uniform_vectors(p);
  return with_k(K, [&](auto k) {
    constexpr int KK = decltype(k)::value;
    if (u) inv_bwd_data_kernel<KK, true><<<grid, kThreads, 0, st>>>(dyb, kb, dxb, p);
    else inv_bwd_data_kernel<KK, false><<<grid, kThreads, 0, st>>>(dyb, kb, dxb, p);
    HB_LAUNCH_CHECK();
    return 0;
  });
}

int hb_involution_bwd_kernel_bf16(const void* x, const void* dy, void* dker, int N, int H, int W, int C, int Cp, int Kp,
                                  int K, int G, int stride, int pad, int dil, void* stream) {
  InvParams p;
  if (int rc = make_params(p, N, H, W, C, Cp, Kp, K, G, stride, pad, dil)) return rc;
  return with_k(K, [&](auto k) {
    return launch_bwd_kernel<decltype(k)::value>((const bf16*)x, (const bf16*)dy, (bf16*)dker, p, (cudaStream_t)stream);
  });
}

}  // extern "C"
