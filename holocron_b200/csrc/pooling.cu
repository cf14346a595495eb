// Blur pooling, global max pooling and Z-pooling (reference holocron/nn/modules/downsample.py:80-99 GlobalMaxPool2d,
// :106-151 BlurPool2d, :170-183 ZPool; holocron/nn/functional.py:139-147 z_pool) over NHWC tensors of bf16 or fp32
// storage, fp32 accumulation. The row pitch Cp is a multiple of one 16-byte vector (8 bf16 or 4 fp32 channels) and
// the logical channel count C is passed separately: channels C..Cp-1 of every output and input gradient are written
// as zeros, whatever the padded inputs hold.
//
// Blur pooling: y[n, oy, ox, c] = sum_{i,j} w[i][j] * x[n, r(oy*s - p + i), r(ox*s - p + j), c] with r() the reflection
// of ReflectionPad2d(p) folded into the index arithmetic (p < H, W: one reflection suffices), so no padded copy of x
// is made. The backward pass is the gather form of the adjoint: a pixel h collects the taps of every padded position
// that reflects onto it (h itself, -h when 1 <= h <= p, 2(H-1) - h when it lies in the bottom pad).
//
// Max / mean reductions: the "mid" kernels reduce the middle axis of an [A, L, M] view (global max pooling: A = N,
// L = H*W, M = Cp; z_pool over H: A = N, L = H, M = W*Cp; over W: A = N*H, L = W, M = Cp), the "last" kernels the
// contiguous channel axis of [R, Cp] rows (z_pool over C). The max keeps its int32 index for the backward pass, which
// writes dx once: dmax at the saved index plus dmean / L everywhere. The order is "NaN first, then larger, then lower
// index", so ties and NaNs route the gradient as torch's max(dim).indices does. Partial results are combined in a
// fixed order (no atomics): every run gives the same bits. Nothing here synchronises with the host.
#include "nhwc.cuh"

namespace {

using namespace hb;
using bf16 = __nv_bfloat16;

constexpr int kThreads = 256;
constexpr int kMaxTaps = 7;

struct BlurParams {
  int N, H, W, C, Cp, Ho, Wo, K, stride, pad;
  float w[kMaxTaps * kMaxTaps];   // the 2-D filter, row-major (kernel parameter space: indexed without local memory)
};

__device__ __forceinline__ int reflect(int t, int n) { return t < 0 ? -t : (t >= n ? 2 * (n - 1) - t : t); }

// One CTA per output row (n, oy); its threads walk the Wo x Cp/V vectors of that row.
template <typename T, int K>
__global__ void __launch_bounds__(kThreads) blur_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, BlurParams p) {
  constexpr int V = Vec16<T>::N;
  const int n = blockIdx.x / p.Ho, oy = blockIdx.x % p.Ho;
  const int cv = p.Cp / V;
  int rows[K];
#pragma unroll
  for (int i = 0; i < K; ++i) rows[i] = reflect(oy * p.stride - p.pad + i, p.H);
  const T* xn = x + (size_t)n * p.H * p.W * p.Cp;
  T* yr = y + ((size_t)n * p.Ho + oy) * p.Wo * p.Cp;
  for (int e = threadIdx.x; e < p.Wo * cv; e += blockDim.x) {
    const int cvec = e % cv, ox = e / cv;
    int cols[K];
#pragma unroll
    for (int j = 0; j < K; ++j) cols[j] = reflect(ox * p.stride - p.pad + j, p.W);
    float acc[V];
#pragma unroll
    for (int l = 0; l < V; ++l) acc[l] = 0.f;
#pragma unroll
    for (int i = 0; i < K; ++i) {
      const T* xr = xn + (size_t)rows[i] * p.W * p.Cp + cvec * V;
#pragma unroll
      for (int j = 0; j < K; ++j) {
        const Vec16<T> v = ld16(xr + (size_t)cols[j] * p.Cp);
        const float wt = p.w[i * K + j];
#pragma unroll
        for (int l = 0; l < V; ++l) acc[l] = fmaf(wt, to_f(v.v[l]), acc[l]);
      }
    }
    st16(yr + (size_t)ox * p.Cp + cvec * V, pack<T>(acc, cvec * V, p.C));
  }
}

// The padded position (in padded coordinates tp = t + pad) of the a-th source of pixel h, or -1 when it has none:
// a = 0 is h itself, a = 1 its mirror in the leading pad (-h), a = 2 its mirror in the trailing pad (2(H-1) - h).
__device__ __forceinline__ int source(int a, int h, int H, int pad) {
  if (a == 0) return h + pad;
  if (a == 1) return (h >= 1 && h <= pad) ? pad - h : -1;
  const int t = 2 * (H - 1) - h;
  return (h <= H - 2 && t <= H - 1 + pad) ? t + pad : -1;
}

// Data gradient, gather form: one CTA per input row (n, h); dx[n, h, w, c] = sum of w[i][j] * dy[n, oy, ox, c] over
// every source (tp, tq) of (h, w) and every tap with oy * s + i = tp, ox * s + j = tq (i = tp mod s, tp mod s + s, ...,
// so no tap is tested for divisibility). Each element is written once.
template <typename T, int K>
__global__ void __launch_bounds__(kThreads) blur_bwd_kernel(const T* __restrict__ dy, T* __restrict__ dx, BlurParams p) {
  constexpr int V = Vec16<T>::N;
  const int n = blockIdx.x / p.H, h = blockIdx.x % p.H;
  const int cv = p.Cp / V;
  const T* dyn = dy + (size_t)n * p.Ho * p.Wo * p.Cp;
  T* dxr = dx + ((size_t)n * p.H + h) * p.W * p.Cp;
  for (int e = threadIdx.x; e < p.W * cv; e += blockDim.x) {
    const int cvec = e % cv, w = e / cv;
    float acc[V];
#pragma unroll
    for (int l = 0; l < V; ++l) acc[l] = 0.f;
#pragma unroll 1
    for (int a = 0; a < 3; ++a) {
      const int tp = source(a, h, p.H, p.pad);
      if (tp < 0) continue;
#pragma unroll 1
      for (int i = tp % p.stride, oy = tp / p.stride; i < K && oy >= 0; i += p.stride, --oy) {
        if (oy >= p.Ho) continue;
        const T* dyr = dyn + (size_t)oy * p.Wo * p.Cp + cvec * V;
#pragma unroll 1
        for (int b = 0; b < 3; ++b) {
          const int tq = source(b, w, p.W, p.pad);
          if (tq < 0) continue;
#pragma unroll 1
          for (int j = tq % p.stride, ox = tq / p.stride; j < K && ox >= 0; j += p.stride, --ox) {
            if (ox >= p.Wo) continue;
            const Vec16<T> g = ld16(dyr + (size_t)ox * p.Cp);
            const float wt = p.w[i * K + j];
#pragma unroll
            for (int l = 0; l < V; ++l) acc[l] = fmaf(wt, to_f(g.v[l]), acc[l]);
          }
        }
      }
    }
    st16(dxr + (size_t)w * p.Cp + cvec * V, pack<T>(acc, cvec * V, p.C));
  }
}

struct MidParams {
  int A, L, M, C, Cp, with_mean;
};

// Middle-axis reduction of x [A, L, M]: CTA (a, slab) owns nv consecutive vectors of M; its kThreads / nv row groups
// scan the rows l = part, part + parts, ... and a fixed tree over the groups combines them. Writes y[a][0][m] = max
// (and y[a][1][m] = mean when with_mean) and idx[a][m].
template <typename T>
__global__ void __launch_bounds__(kThreads) mid_fwd_kernel(const T* __restrict__ x, T* __restrict__ y,
                                                           int* __restrict__ idx, MidParams p, int nv) {
  constexpr int V = Vec16<T>::N;
  __shared__ float s_max[kThreads][V];
  __shared__ float s_sum[kThreads][V];
  __shared__ int s_idx[kThreads][V];
  const int a = blockIdx.x;
  const int vi = threadIdx.x % nv, part = threadIdx.x / nv, parts = kThreads / nv;
  const int mv = blockIdx.y * nv + vi;
  const bool live = mv < p.M / V;
  float mx[V], sm[V];
  int ix[V];
#pragma unroll
  for (int l = 0; l < V; ++l) {
    mx[l] = -INFINITY;
    sm[l] = 0.f;
    ix[l] = kNoIndex;
  }
  if (live) {
    const T* xa = x + (size_t)a * p.L * p.M + (size_t)mv * V;
#pragma unroll 4
    for (int r = part; r < p.L; r += parts) {
      const Vec16<T> v = ld16(xa + (size_t)r * p.M);
#pragma unroll
      for (int l = 0; l < V; ++l) {
        const float f = to_f(v.v[l]);
        if (better(f, r, mx[l], ix[l])) {
          mx[l] = f;
          ix[l] = r;
        }
        sm[l] += f;
      }
    }
  }
#pragma unroll
  for (int l = 0; l < V; ++l) {
    s_max[threadIdx.x][l] = mx[l];
    s_sum[threadIdx.x][l] = sm[l];
    s_idx[threadIdx.x][l] = ix[l];
  }
  __syncthreads();
  for (int half = parts / 2; half > 0; half /= 2) {
    if (part < half) {
      const int o = threadIdx.x + half * nv;
#pragma unroll
      for (int l = 0; l < V; ++l) {
        if (better(s_max[o][l], s_idx[o][l], mx[l], ix[l])) {
          mx[l] = s_max[o][l];
          ix[l] = s_idx[o][l];
        }
        sm[l] += s_sum[o][l];
        s_max[threadIdx.x][l] = mx[l];
        s_idx[threadIdx.x][l] = ix[l];
        s_sum[threadIdx.x][l] = sm[l];
      }
    }
    __syncthreads();
  }
  if (part != 0 || !live) return;
  const int c0 = (mv * V) % p.Cp;
  float mean[V];
#pragma unroll
  for (int l = 0; l < V; ++l) mean[l] = sm[l] / (float)p.L;
  T* ya = y + (size_t)a * (p.with_mean ? 2 : 1) * p.M + (size_t)mv * V;
  st16(ya, pack<T, true>(mx, c0, p.C));
  if (p.with_mean) st16(ya + p.M, pack<T>(mean, c0, p.C));
  int* ia = idx + (size_t)a * p.M + (size_t)mv * V;
#pragma unroll
  for (int l = 0; l < V; ++l) ia[l] = c0 + l < p.C ? ix[l] : 0;
}

// dx[a, l, m] = (l == idx[a, m] ? dmax : 0) + dmean / L, one vector per step. I is the index type: 32-bit whenever the
// vector count allows it (the decomposition is the costliest part of this write-only pass).
template <typename T, typename I>
__global__ void __launch_bounds__(kThreads) mid_bwd_kernel(const T* __restrict__ dy, const int* __restrict__ idx,
                                                           T* __restrict__ dx, MidParams p) {
  constexpr int V = Vec16<T>::N;
  const I mvs = (I)(p.M / V);
  const I total = (I)p.A * (I)p.L * mvs;
  for (I e = (I)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (I)gridDim.x * blockDim.x) {
    const I mv = e % mvs, row = e / mvs;
    const int r = (int)(row % (I)p.L);
    const size_t a = (size_t)(row / (I)p.L);
    const size_t m0 = (size_t)mv * V;
    const int c0 = (int)(m0 % (size_t)p.Cp);
    const Vec16<T> gmax = ld16(dy + a * (p.with_mean ? 2 : 1) * p.M + m0);
    Vec16<T> gmean;
    if (p.with_mean) gmean = ld16(dy + (a * 2 + 1) * p.M + m0);
    const int4* ia = reinterpret_cast<const int4*>(idx + a * p.M + m0);   // V indices, 16-byte aligned
    int hit[V];
#pragma unroll
    for (int q = 0; q < V / 4; ++q) {
      const int4 iv = ia[q];
      hit[4 * q] = iv.x; hit[4 * q + 1] = iv.y; hit[4 * q + 2] = iv.z; hit[4 * q + 3] = iv.w;
    }
    float g[V];
#pragma unroll
    for (int l = 0; l < V; ++l) {
      float v = p.with_mean ? to_f(gmean.v[l]) / (float)p.L : 0.f;
      if (hit[l] == r) v = to_f(gmax.v[l]) + v;
      g[l] = v;
    }
    st16(dx + (size_t)e * V, pack<T>(g, c0, p.C));
  }
}

// Channel-axis reduction of x [R, Cp] over the logical C channels: a group of g lanes (a power of two up to 32) per
// row, each scanning vectors v = lane, lane + g, ..., combined by an xor butterfly (every lane ends with the same
// bits). Writes y[r][0] = max, y[r][1] = mean and idx[r].
template <typename T>
__global__ void __launch_bounds__(kThreads) last_fwd_kernel(const T* __restrict__ x, T* __restrict__ y,
                                                            int* __restrict__ idx, int R, int C, int Cp, int g) {
  constexpr int V = Vec16<T>::N;
  const int lane = threadIdx.x % g;
  const int rows_per_cta = kThreads / g;
  const long long r = (long long)blockIdx.x * rows_per_cta + threadIdx.x / g;
  const bool live = r < R;
  float mx = -INFINITY, sm = 0.f;
  int ix = kNoIndex;
  if (live) {
    const T* xr = x + (size_t)r * Cp;
    for (int v = lane; v * V < C; v += g) {
      const Vec16<T> xv = ld16(xr + v * V);
#pragma unroll
      for (int l = 0; l < V; ++l) {
        const int c = v * V + l;
        if (c >= C) break;
        const float f = to_f(xv.v[l]);
        if (better(f, c, mx, ix)) {
          mx = f;
          ix = c;
        }
        sm += f;
      }
    }
  }
  group_max_sum(mx, ix, sm, g);
  if (!live || lane != 0) return;
  y[(size_t)r * 2] = same_bits<T>(mx);
  y[(size_t)r * 2 + 1] = from_f<T>(sm / (float)C);
  idx[r] = ix;
}

template <typename T, typename I>
__global__ void __launch_bounds__(kThreads) last_bwd_kernel(const T* __restrict__ dy, const int* __restrict__ idx,
                                                            T* __restrict__ dx, int R, int C, int Cp) {
  constexpr int V = Vec16<T>::N;
  const I cv = (I)(Cp / V);
  const I total = (I)R * cv;
  for (I e = (I)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (I)gridDim.x * blockDim.x) {
    const I r = e / cv;
    const int c0 = (int)(e % cv) * V;
    const float gmax = to_f(dy[(size_t)r * 2]);
    const float gmean = to_f(dy[(size_t)r * 2 + 1]) / (float)C;
    const int hit = idx[r];
    float g[V];
#pragma unroll
    for (int l = 0; l < V; ++l) g[l] = c0 + l == hit ? gmax + gmean : gmean;
    st16(dx + (size_t)e * V, pack<T>(g, c0, C));
  }
}

// 0 when the shape is supported (fills p), otherwise cudaErrorInvalidValue
int make_blur(BlurParams& p, const float* taps, int N, int H, int W, int C, int Cp, int K, int stride, int dtype) {
  if (bad_rows(C, Cp, dtype) || N <= 0 || H <= 0 || W <= 0 || K < 2 || K > kMaxTaps || stride < 1 || taps == nullptr)
    return (int)cudaErrorInvalidValue;
  p.N = N; p.H = H; p.W = W; p.C = C; p.Cp = Cp; p.K = K; p.stride = stride;
  p.pad = ((stride - 1) + (K - 1)) / 2;
  if (p.pad >= H || p.pad >= W) return (int)cudaErrorInvalidValue;   // ReflectionPad2d's own limit
  if (!window_out(H, K, stride, p.pad, 1, p.Ho) || !window_out(W, K, stride, p.pad, 1, p.Wo) ||
      (long long)N * H >= 0x7fffffffLL || (long long)N * p.Ho >= 0x7fffffffLL)
    return (int)cudaErrorInvalidValue;
  for (int t = 0; t < K * K; ++t) p.w[t] = taps[t];
  return 0;
}

template <typename T>
int launch_blur(bool fwd, const void* in, void* out, const BlurParams& p, cudaStream_t st) {
  const T* a = (const T*)in;
  T* b = (T*)out;
  const unsigned grid = (unsigned)(fwd ? p.N * p.Ho : p.N * p.H);
#define HB_BLUR_CASE(KK)                                                           \
  case KK:                                                                         \
    if (fwd) blur_fwd_kernel<T, KK><<<grid, kThreads, 0, st>>>(a, b, p);           \
    else blur_bwd_kernel<T, KK><<<grid, kThreads, 0, st>>>(a, b, p);               \
    break;
  switch (p.K) {
    HB_BLUR_CASE(2)
    HB_BLUR_CASE(3)
    HB_BLUR_CASE(4)
    HB_BLUR_CASE(5)
    HB_BLUR_CASE(6)
    HB_BLUR_CASE(7)
    default: return (int)cudaErrorInvalidValue;
  }
#undef HB_BLUR_CASE
  HB_LAUNCH_CHECK();
  return 0;
}

int make_mid(MidParams& p, int A, int L, int M, int C, int Cp, int with_mean, int dtype) {
  if (bad_rows(C, Cp, dtype) || A <= 0 || L <= 0 || M <= 0 || M % Cp != 0) return (int)cudaErrorInvalidValue;
  if ((M / vec_width(dtype) + 31) / 32 > 65535) return (int)cudaErrorInvalidValue;   // grid.y slabs of nv <= 32 vectors
  p = MidParams{A, L, M, C, Cp, with_mean ? 1 : 0};
  return 0;
}

template <typename T>
int launch_mid_fwd(const void* x, void* y, int* idx, const MidParams& p, cudaStream_t st) {
  constexpr int V = Vec16<T>::N;
  // up to 32 vectors (512 contiguous bytes) across a CTA, the other threads split the rows
  const int nv = pow2_at_least(p.M / V, 32);
  const dim3 grid((unsigned)p.A, (unsigned)((p.M / V + nv - 1) / nv));
  mid_fwd_kernel<T><<<grid, kThreads, 0, st>>>((const T*)x, (T*)y, idx, p, nv);
  HB_LAUNCH_CHECK();
  return 0;
}

template <typename T>
int launch_mid_bwd(const void* dy, const int* idx, void* dx, const MidParams& p, cudaStream_t st) {
  constexpr int V = Vec16<T>::N;
  const size_t total = (size_t)p.A * p.L * (p.M / V);
  const int grid = stream_grid(total, kThreads, 16);
  if (total + (size_t)grid * kThreads < 0xffffffffull)
    mid_bwd_kernel<T, unsigned><<<grid, kThreads, 0, st>>>((const T*)dy, idx, (T*)dx, p);
  else
    mid_bwd_kernel<T, unsigned long long><<<grid, kThreads, 0, st>>>((const T*)dy, idx, (T*)dx, p);
  HB_LAUNCH_CHECK();
  return 0;
}

template <typename T>
int launch_last(bool fwd, const void* in, void* out, int* idx, int R, int C, int Cp, cudaStream_t st) {
  constexpr int V = Vec16<T>::N;
  if (fwd) {
    const int g = lane_group((C + V - 1) / V);
    const unsigned grid = (unsigned)(((long long)R * g + kThreads - 1) / kThreads);
    last_fwd_kernel<T><<<grid, kThreads, 0, st>>>((const T*)in, (T*)out, idx, R, C, Cp, g);
  } else {
    const size_t total = (size_t)R * (Cp / V);
    const int grid = stream_grid(total, kThreads, 16);
    if (total + (size_t)grid * kThreads < 0xffffffffull)
      last_bwd_kernel<T, unsigned><<<grid, kThreads, 0, st>>>((const T*)in, idx, (T*)out, R, C, Cp);
    else
      last_bwd_kernel<T, unsigned long long><<<grid, kThreads, 0, st>>>((const T*)in, idx, (T*)out, R, C, Cp);
  }
  HB_LAUNCH_CHECK();
  return 0;
}

bool bad_last(int R, int C, int Cp, int dtype) { return bad_rows(C, Cp, dtype) || R <= 0; }

}  // namespace

extern "C" {

int hb_blurpool_fwd(const void* x, void* y, const float* taps, int N, int H, int W, int C, int Cp, int K, int stride,
                    int dtype, void* stream) {
  BlurParams p;
  if (int rc = make_blur(p, taps, N, H, W, C, Cp, K, stride, dtype)) return rc;
  return with_dtype(dtype, [&](auto t) { return launch_blur<decltype(t)>(true, x, y, p, (cudaStream_t)stream); });
}

int hb_blurpool_bwd(const void* dy, void* dx, const float* taps, int N, int H, int W, int C, int Cp, int K, int stride,
                    int dtype, void* stream) {
  BlurParams p;
  if (int rc = make_blur(p, taps, N, H, W, C, Cp, K, stride, dtype)) return rc;
  return with_dtype(dtype, [&](auto t) { return launch_blur<decltype(t)>(false, dy, dx, p, (cudaStream_t)stream); });
}

int hb_pool_mid_fwd(const void* x, void* y, int* idx, int A, int L, int M, int C, int Cp, int with_mean, int dtype,
                    void* stream) {
  MidParams p;
  if (int rc = make_mid(p, A, L, M, C, Cp, with_mean, dtype)) return rc;
  return with_dtype(dtype, [&](auto t) { return launch_mid_fwd<decltype(t)>(x, y, idx, p, (cudaStream_t)stream); });
}

int hb_pool_mid_bwd(const void* dy, const int* idx, void* dx, int A, int L, int M, int C, int Cp, int with_mean,
                    int dtype, void* stream) {
  MidParams p;
  if (int rc = make_mid(p, A, L, M, C, Cp, with_mean, dtype)) return rc;
  return with_dtype(dtype, [&](auto t) { return launch_mid_bwd<decltype(t)>(dy, idx, dx, p, (cudaStream_t)stream); });
}

int hb_pool_last_fwd(const void* x, void* y, int* idx, int R, int C, int Cp, int dtype, void* stream) {
  if (bad_last(R, C, Cp, dtype)) return (int)cudaErrorInvalidValue;
  return with_dtype(dtype, [&](auto t) {
    return launch_last<decltype(t)>(true, x, y, idx, R, C, Cp, (cudaStream_t)stream);
  });
}

int hb_pool_last_bwd(const void* dy, const int* idx, void* dx, int R, int C, int Cp, int dtype, void* stream) {
  if (bad_last(R, C, Cp, dtype)) return (int)cudaErrorInvalidValue;
  return with_dtype(dtype, [&](auto t) {
    return launch_last<decltype(t)>(false, dy, dx, (int*)idx, R, C, Cp, (cudaStream_t)stream);
  });
}

}  // extern "C"
