// Classification / segmentation losses: focal, poly-1 (hard + soft targets; with eps = 0 also the multi-label cross
// entropy), dice, complement cross entropy and the mutual channel loss.
// Reference: holocron/nn/functional.py:59-113 (focal_loss), :540-613 (poly_loss), :503-537 (dice_loss),
// :150-191 (multilabel_cross_entropy), :194-255 (complement_cross_entropy), :258-319 (mutual_channel_loss).
//
// Logits are [N, K, S] (S = product of the spatial dims, possibly 1); a "position" is one (n, s) pair.
// The reference runs log_softmax + transpose/flatten/gather + boolean-mask indexing + mean (~10 kernels, 4-6
// passes over N*K and a host sync for the mask). Here: ONE pass over the logits produces the per-position
// loss and per-CTA partial sums (fp64, combined in a fixed order -> deterministic), and the backward pass
// recomputes the softmax and writes dlogits in one more pass.
//   S == 1 : one warp per position, lanes stride over the K classes (coalesced rows)
//   S  > 1 : one thread per position, consecutive threads = consecutive s (coalesced for every class k)
#include <type_traits>

#include "common.cuh"

namespace {

using namespace hb;

constexpr int kThreads = 256;

enum LossKind { FOCAL = 0, POLY = 1 };

// The arguments of the class-axis kernels (focal / poly-1 with hard or soft targets, complement cross entropy).
struct LossParams {
  const void* x;            // [N, K, S]
  const long long* target;  // [N, S] class indices (int64)          (hard targets, complement CE)
  const void* soft;         // [N, K, S] soft targets, same dtype    (soft targets)
  const float* weight;      // [K] or null
  float* loss_pos;          // forward: [N*S] per-position loss
  double* partials;         // forward: [grid][2 or 3] per-block partial sums (see finalize_kernel)
  const float* gout;        // backward: reduction none: [N*S]; else 1 element
  const float* fwd_out;     // backward: {sum, count, mean} of the forward (count used for 'mean')
  void* dx;                 // backward: [N, K, S]
  int N, K, S;
  int ignore_index;         // class column: honoured only when 0 <= ignore_index < K (reference quirk)
  int kind;                 // LossKind (hard targets)
  int reduction;            // backward: 0 none, 1 mean, 2 sum
  float gamma;              // focal exponent / complement-term weight
  float eps;                // poly-1 epsilon
};

// The gradient scale of one position's term: gout[pos] for 'none', gout[0] for 'sum' and gout[0] / den for 'mean', where
// den is the forward's count *count for a term averaged over its counted positions, or the number of positions P when
// count is null. `reduced` is the 'mean' / 'sum' value, the same for every position.
struct GradScale {
  const float* gout;
  int reduction;
  float reduced;
  // `dropped`: a position left out of the count gets no share of a 'mean' / 'sum' gradient
  __device__ __forceinline__ float at(long long pos, bool dropped = false) const {
    return reduction == 0 ? gout[pos] : (dropped ? 0.f : reduced);
  }
};
__device__ __forceinline__ GradScale grad_scale(const float* gout, int reduction, const float* count, long long P) {
  const float reduced = reduction == 0 ? 0.f : (reduction == 1 ? gout[0] / (count ? *count : (float)P) : gout[0]);
  return {gout, reduction, reduced};
}

// Block-wide sums of this thread's partials, stored as partials[NP * block + i] (NP = number of values), which
// finalize_kernel folds in block order.
template <class... D>
__device__ __forceinline__ void store_partials(double* partials, double* red, D... v) {
  constexpr int NP = sizeof...(D);
  const double s[NP] = {block_sum<double>(v, red)...};
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 0; i < NP; ++i) partials[NP * blockIdx.x + i] = s[i];
  }
}

// grid-stride iterations of the thread that starts at item i0 < stride: the soft-target kernels count their positions
// from it after the loop, so the count needs no accumulator while the loop runs
__device__ __forceinline__ double thread_iters(long long i0, long long total, long long stride) {
  return i0 < total ? (double)((total - 1 - i0) / stride + 1) : 0.0;
}

// partials [n][NP] = {A, B, C} (NP = 3) or {A, B} (NP = 2, C = 0): A is the (weighted) sum of the per-position terms
// counted by B; C a second term averaged over all P positions. out = {A + coef * C, B, A / B + coef * C / P} (with
// C = 0: {A, B, A / B}), each summed in block order. One warp: lane u loads block i0 + u (32 blocks per round trip to L2)
// and the sums take the blocks in order through shuffles.
template <int NP>
__global__ void finalize_kernel(const double* partials, int n, double P, float coef, float* out) {
  const int lane = threadIdx.x & 31;
  double s[3] = {0.0, 0.0, 0.0};
  for (int i0 = 0; i0 < n; i0 += 32) {
    double v[NP];
#pragma unroll
    for (int j = 0; j < NP; ++j) v[j] = i0 + lane < n ? partials[NP * (i0 + lane) + j] : 0.0;
    const int m = n - i0 < 32 ? n - i0 : 32;
    for (int u = 0; u < m; ++u) {
#pragma unroll
      for (int j = 0; j < NP; ++j) s[j] += __shfl_sync(0xffffffffu, v[j], u);
    }
  }
  if (lane == 0) {
    out[0] = (float)(s[0] + (double)coef * s[2]);
    out[1] = (float)s[1];
    out[2] = (float)(s[0] / s[1] + (double)coef * s[2] / P);
  }
}

// k-loop shapes: one thread owns a position (S > 1) or a warp does, its lanes striding over the classes (S == 1)
struct ThreadLanes {
  static constexpr int kStep = 1;
  int k0 = 0;
  __device__ float max(float v) const { return v; }
  __device__ float sum(float v) const { return v; }
};
struct WarpLanes {
  static constexpr int kStep = 32;
  int k0;
  __device__ float max(float v) const { return warp_max(v); }
  __device__ float sum(float v) const { return warp_sum(v); }
};

// Calls f(ln, xp, dp, st, pos) for each of this thread's positions: xp / dp point at the position's class 0 in x / dx and
// st is the class stride. S == 1: a warp per position (WarpLanes over a contiguous row); S > 1: a thread per position.
template <typename T, class F>
__device__ __forceinline__ void for_each_position(const LossParams& p, F f) {
  const T* x = (const T*)p.x;
  T* dx = (T*)p.dx;
  const long long P = (long long)p.N * p.S;
  if (p.S == 1) {
    const WarpLanes ln{threadIdx.x & 31};
    const long long warps = (long long)gridDim.x * (kThreads / 32);
    for (long long pos = (long long)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5); pos < P; pos += warps)
      f(ln, x + pos * p.K, dx + pos * p.K, 1LL, pos);
  } else {
    const ThreadLanes ln{};
    const long long stride = (long long)gridDim.x * kThreads;
    for (long long pos = (long long)blockIdx.x * kThreads + threadIdx.x; pos < P; pos += stride) {
      const long long off = (pos / p.S) * p.K * p.S + pos % p.S;
      f(ln, x + off, dx + off, (long long)p.S, pos);
    }
  }
}

// log sum_k exp(x_k) of one position, x_at(k) being class k
template <class Ln, class X>
__device__ __forceinline__ float lane_lse(const Ln& ln, X x_at, int K) {
  float mx = -INFINITY;
  for (int k = ln.k0; k < K; k += Ln::kStep) mx = fmaxf(mx, x_at(k));
  mx = ln.max(mx);
  float s = 0.f;
  for (int k = ln.k0; k < K; k += Ln::kStep) s += expf(x_at(k) - mx);
  s = ln.sum(s);
  return mx + logf(s);
}

// (1 - pt)^gamma: gamma = 2 (the default) and 1 are plain products - what torch.pow does for those exponents too - so the
// ~100-instruction powf only runs for other exponents
__device__ __forceinline__ float focal_mod(float om, float gamma) {
  if (gamma == 2.f) return om * om;
  if (gamma == 1.f) return om;
  return gamma == 0.f ? 1.f : powf(om, gamma);
}
__device__ __forceinline__ float hard_loss(const LossParams& p, float logpt, float w) {
  const float pt = expf(logpt);
  if (p.kind == FOCAL) {
    const float mod = focal_mod(fmaxf(1.f - pt, 0.f), p.gamma);
    return -mod * (w * logpt);
  }
  return w * (-logpt + p.eps * (1.f - pt));
}
// d loss / d logpt
__device__ __forceinline__ float hard_dloss(const LossParams& p, float logpt, float w) {
  const float pt = expf(logpt);
  if (p.kind == FOCAL) {
    const float om = fmaxf(1.f - pt, 0.f);
    if (p.gamma == 0.f) return -w;
    const float mod = focal_mod(om, p.gamma);
    const float dmod = om > 0.f ? p.gamma * focal_mod(om, p.gamma - 1.f) * pt : 0.f;  // -(d mod / d logpt)
    return -w * (mod - dmod * logpt);
  }
  return w * (-1.f - p.eps * pt);
}

// ---- hard targets ---------------------------------------------------------------------------------
template <typename T, bool kBackward, class Ln>
__device__ __forceinline__ void hard_position(const LossParams& p, const Ln& ln, const T* xp, T* dp, long long st,
                                              long long pos, double& lsum, double& lcnt) {
  auto x_at = [&](int k) { return to_f(xp[k * st]); };
  const float lse = lane_lse(ln, x_at, p.K);
  const long long t = p.target[pos];
  const bool inr = t >= 0 && t < p.K;
  const bool skip = p.ignore_index >= 0 && p.ignore_index < p.K && t == p.ignore_index;
  if (!kBackward) {
    float l = NAN;
    if (inr) l = hard_loss(p, x_at((int)t) - lse, p.weight ? p.weight[t] : 1.f);
    if (ln.k0 == 0) {
      p.loss_pos[pos] = l;
      if (!skip) { lsum += l; lcnt += 1.0; }
    }
  } else {
    float c = 0.f;
    if (inr) c = grad_scale(p.gout, p.reduction, p.fwd_out + 1, 0).at(pos, skip) * hard_dloss(p, x_at((int)t) - lse, p.weight ? p.weight[t] : 1.f);
    for (int k = ln.k0; k < p.K; k += Ln::kStep) {
      const float pk = expf(x_at(k) - lse);
      dp[k * st] = from_f<T>(c * ((k == t ? 1.f : 0.f) - pk));
    }
  }
}

template <typename T, bool kBackward>
__global__ void __launch_bounds__(kThreads) hard_kernel(LossParams p) {
  __shared__ double red[32];
  double lsum = 0.0, lcnt = 0.0;
  for_each_position<T>(p, [&](const auto& ln, const T* xp, T* dp, long long st, long long pos) {
    hard_position<T, kBackward>(p, ln, xp, dp, st, pos, lsum, lcnt);
  });
  if (!kBackward) store_partials(p.partials, red, lsum, lcnt);
}

// ---- poly loss with soft targets ------------------------------------------------------------------
// per position: L = sum_{k valid} w_k * (-z_k + eps * (1 - exp(z_k))),  z_k = log_softmax(x)_k * t_k
// One thread per position at every S. The second partial counts the positions, so the finalize gives {sum, P, sum / P}.
template <typename T, bool kBackward>
__global__ void __launch_bounds__(kThreads) poly_soft_kernel(LossParams p) {
  __shared__ double red[32];
  const T* x = (const T*)p.x;
  const T* tg = (const T*)p.soft;
  T* dx = (T*)p.dx;
  const long long P = (long long)p.N * p.S;
  const bool ign = p.ignore_index >= 0 && p.ignore_index < p.K;
  double lsum = 0.0;
  const ThreadLanes ln{};
  const long long stride = (long long)gridDim.x * kThreads, pos0 = (long long)blockIdx.x * kThreads + threadIdx.x;
  for (long long pos = pos0; pos < P; pos += stride) {
    const long long n = pos / p.S, s = pos % p.S;
    const long long off = n * p.K * p.S + s;
    auto x_at = [&](int k) { return to_f(x[off + (long long)k * p.S]); };
    const float lse = lane_lse(ln, x_at, p.K);
    if (!kBackward) {
      float l = 0.f;
      for (int k = 0; k < p.K; ++k) {
        if (ign && k == p.ignore_index) continue;
        const float z = (x_at(k) - lse) * to_f(tg[off + (long long)k * p.S]);
        l += (p.weight ? p.weight[k] : 1.f) * (-z + p.eps * (1.f - expf(z)));
      }
      p.loss_pos[pos] = l;
      lsum += l;
    } else {
      const float g = grad_scale(p.gout, p.reduction, nullptr, P).at(pos);
      // dL/dx_j = c_j t_j - p_j * sum_k c_k t_k,   c_k = w_k * valid_k * (-1 - eps * exp(z_k))
      float tot = 0.f;
      for (int k = 0; k < p.K; ++k) {
        if (ign && k == p.ignore_index) continue;
        const float tk = to_f(tg[off + (long long)k * p.S]);
        const float z = (x_at(k) - lse) * tk;
        tot += (p.weight ? p.weight[k] : 1.f) * (-1.f - p.eps * expf(z)) * tk;
      }
      for (int k = 0; k < p.K; ++k) {
        const float lp = x_at(k) - lse;
        float ck = 0.f;
        if (!(ign && k == p.ignore_index)) {
          const float tk = to_f(tg[off + (long long)k * p.S]);
          ck = (p.weight ? p.weight[k] : 1.f) * (-1.f - p.eps * expf(lp * tk)) * tk;
        }
        dx[off + (long long)k * p.S] = from_f<T>(g * (ck - expf(lp) * tot));
      }
    }
  }
  if (!kBackward) store_partials(p.partials, red, lsum, thread_iters(pos0, P, stride));
}

int grid_for(long long work, int per_block) {
  long long g = (work + per_block - 1) / per_block;
  if (g < 1) g = 1;
  if (g > HB_NUM_SMS * 8) g = HB_NUM_SMS * 8;
  return (int)g;
}


// ---- S > 1, K <= 32: register-resident class columns -----------------------------------------------
// The one-thread-per-position kernels above read a 2- or 4-byte element per load and pass over the K classes two or
// three times: too few bytes in flight to stream at the HBM rate. Here a thread owns V = 8 /
// sizeof(T) consecutive positions, issues its K 8-byte loads back to back into registers (KMAX of them, -inf beyond
// K) and computes max, sum of exponentials, the target logit and - backward - the gradient from those registers:
// the logits are read from HBM exactly once and every store is a full 8-byte (logits) / 16-byte (fp32 loss) vector.
// exp(x) for x <= 0 on the MUFU unit: one FMUL + ex2.approx.ftz (flush-to-zero: results below 2^-126 are 0 either way here)
__device__ __forceinline__ float exp_mufu(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x * 1.4426950408889634f));
  return y;
}

// exp(x - m) for x <= m as ex2((x - m) * log2e): x - m is exact wherever the term matters (Sterbenz), so the argument's
// error scales with |x - m| as in expf(x - m). Folding m into an FFMA, ex2(x * log2e - m * log2e), saves one instruction
// but rounds m * log2e, an error that grows with the largest logit: 4e-5 relative at logits near 1000.
constexpr float kLog2e = 1.4426950408889634f;
__device__ __forceinline__ float exp_shift(float x, float m) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"((x - m) * kLog2e));
  return y;
}
template <typename T> __device__ __forceinline__ T neg_inf();
template <> __device__ __forceinline__ float neg_inf<float>() { return -INFINITY; }
template <> __device__ __forceinline__ __nv_bfloat16 neg_inf<__nv_bfloat16>() { return __ushort_as_bfloat16((unsigned short)0xFF80); }
template <> __device__ __forceinline__ __half neg_inf<__half>() { return __ushort_as_half((unsigned short)0xFC00); }

template <typename T> struct Vec8 {
  static constexpr int N = 8 / sizeof(T);
  union { uint2 raw; T v[N]; };
};
template <typename T> __device__ __forceinline__ Vec8<T> ld8(const T* p) {
  Vec8<T> r; r.raw = __ldg(reinterpret_cast<const uint2*>(p)); return r;
}
template <typename T> __device__ __forceinline__ void st8(T* p, const Vec8<T>& v) { *reinterpret_cast<uint2*>(p) = v.raw; }

// Instruction diet (the first register-resident version was ISSUE bound at ~45 instructions per logit, no faster than the
// scalar kernels): 32-bit class stride (K * S < 2^31 checked by the launcher) so a class column is one IMAD.WIDE away, int
// targets (one ISETP per logit instead of two), and MUFU.EX2 (exp_mufu) for the per-logit exponentials - arguments are <= 0,
// where its error is ~2 ulp on the terms that matter; the per-position logf / expf / powf stay IEEE.

// The front end of both register-column kernels: the KMAX class columns of the logits at xk (-inf beyond K) into r and,
// with kSoft, of the soft targets at qk (0 beyond K) into q.
template <typename T, int KMAX, bool kSoft>
__device__ __forceinline__ void load_columns(Vec8<T> (&r)[KMAX], Vec8<T>* q, const T* xk, const T* qk, int K,
                                             unsigned S) {
  constexpr int V = Vec8<T>::N;
  // classes k >= K hold -inf: the compute loops run unpredicated over KMAX (exp(-inf) = 0, never the max or the
  // target); two dozen `k < K` predicates kept live across the body made ptxas shuffle them through P2R / R2P
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    if (k < K) {
      r[k] = ld8(xk);
      if constexpr (kSoft) q[k] = ld8(qk);
    } else {
#pragma unroll
      for (int v = 0; v < V; ++v) {
        r[k].v[v] = neg_inf<T>();
        if constexpr (kSoft) q[k].v[v] = from_f<T>(0.f);
      }
    }
    xk += S;
    if constexpr (kSoft) qk += S;
  }
}

// each position's max and sum of exp(x - max) over the columns; visit(k, v, x) sees every logit of the max pass
template <typename T, int KMAX, class Visit>
__device__ __forceinline__ void max_sumexp(const Vec8<T> (&r)[KMAX], float (&mx)[Vec8<T>::N], float (&sum)[Vec8<T>::N],
                                           Visit visit) {
  constexpr int V = Vec8<T>::N;
#pragma unroll
  for (int v = 0; v < V; ++v) { mx[v] = -INFINITY; sum[v] = 0.f; }
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const float f = to_f(r[k].v[v]);
      mx[v] = fmaxf(mx[v], f);
      visit(k, v, f);
    }
  }
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
#pragma unroll
    for (int v = 0; v < V; ++v) sum[v] += exp_shift(to_f(r[k].v[v]), mx[v]);
  }
}

template <typename T, int KMAX, bool kBackward>
__global__ void __launch_bounds__(kThreads) hard_vec_kernel(LossParams p) {
  constexpr int V = Vec8<T>::N;
  __shared__ double red[32];
  const T* x = (const T*)p.x;
  T* dx = (T*)p.dx;
  const int K = p.K;
  const unsigned S = (unsigned)p.S, SV = S / V;
  const long long PV = (long long)p.N * SV;
  const bool ign = p.ignore_index >= 0 && p.ignore_index < K;
  GradScale gs{};
  if (kBackward) gs = grad_scale(p.gout, p.reduction, p.fwd_out + 1, 0);
  double lsum = 0.0, lcnt = 0.0;
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long pv = (long long)blockIdx.x * kThreads + threadIdx.x; pv < PV; pv += stride) {
    const long long n = pv / SV;
    const unsigned s0 = (unsigned)(pv - n * SV) * V;
    Vec8<T> r[KMAX];
    load_columns<T, KMAX, false>(r, nullptr, x + n * K * S + s0, nullptr, K, S);
    int t[V];       // class index, -1 when outside [0, K)
    bool skip[V];   // ignored position
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const long long tl = p.target[n * S + s0 + v];
      t[v] = (tl >= 0 && tl < K) ? (int)tl : -1;
      skip[v] = ign && tl == p.ignore_index;
    }
    float mx[V], sum[V], xt[V];
#pragma unroll
    for (int v = 0; v < V; ++v) xt[v] = 0.f;
    max_sumexp<T, KMAX>(r, mx, sum, [&](int k, int v, float f) { xt[v] = t[v] == k ? f : xt[v]; });
    if (!kBackward) {
#pragma unroll
      for (int v = 0; v < V; ++v) {
        float l = NAN;
        if (t[v] >= 0) l = hard_loss(p, xt[v] - (mx[v] + logf(sum[v])), p.weight ? p.weight[t[v]] : 1.f);
        p.loss_pos[n * S + s0 + v] = l;
        if (!skip[v]) { lsum += l; lcnt += 1.0; }
      }
    } else {
      float lse[V], c[V];
#pragma unroll
      for (int v = 0; v < V; ++v) {
        lse[v] = mx[v] + logf(sum[v]);
        const float g = gs.at(n * S + s0 + v, skip[v]);
        c[v] = 0.f;
        if (t[v] >= 0) c[v] = g * hard_dloss(p, xt[v] - lse[v], p.weight ? p.weight[t[v]] : 1.f);
      }
      T* dp = dx + n * K * S + s0;
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        Vec8<T> o;
#pragma unroll
        for (int v = 0; v < V; ++v) {
          const float pk = exp_shift(to_f(r[k].v[v]), lse[v]);
          o.v[v] = from_f<T>(c[v] * ((t[v] == k ? 1.f : 0.f) - pk));
        }
        if (k < K) st8(dp, o);
        dp += S;
      }
    }
  }
  if (!kBackward) store_partials(p.partials, red, lsum, lcnt);
}

// soft-target poly loss, same layout: logits AND soft targets in registers
template <typename T, int KMAX, bool kBackward>
__global__ void __launch_bounds__(kThreads) poly_soft_vec_kernel(LossParams p) {
  constexpr int V = Vec8<T>::N;
  __shared__ double red[32];
  const T* x = (const T*)p.x;
  const T* tg = (const T*)p.soft;
  T* dx = (T*)p.dx;
  const int K = p.K;
  const unsigned S = (unsigned)p.S, SV = S / V;
  const long long PV = (long long)p.N * SV;
  const bool ign = p.ignore_index >= 0 && p.ignore_index < K;
  double lsum = 0.0;
  const long long stride = (long long)gridDim.x * kThreads, pv0 = (long long)blockIdx.x * kThreads + threadIdx.x;
  for (long long pv = pv0; pv < PV; pv += stride) {
    const long long n = pv / SV;
    const unsigned s0 = (unsigned)(pv - n * SV) * V;
    const long long off = n * K * S + s0;
    Vec8<T> r[KMAX], q[KMAX];
    load_columns<T, KMAX, true>(r, q, x + off, tg + off, K, S);
    float mx[V], sum[V], lse[V];
    max_sumexp<T, KMAX>(r, mx, sum, [](int, int, float) {});
#pragma unroll
    for (int v = 0; v < V; ++v) lse[v] = mx[v] + logf(sum[v]);
    float acc[V];   // forward: the loss; backward: sum_k c_k t_k
#pragma unroll
    for (int v = 0; v < V; ++v) acc[v] = 0.f;
#pragma unroll
    for (int k = 0; k < KMAX; ++k)
      if (k < K && !(ign && k == p.ignore_index)) {
        const float w = p.weight ? p.weight[k] : 1.f;
#pragma unroll
        for (int v = 0; v < V; ++v) {
          const float tk = to_f(q[k].v[v]);
          const float z = (to_f(r[k].v[v]) - lse[v]) * tk;
          if (!kBackward) acc[v] += w * (-z + p.eps * (1.f - exp_mufu(z)));
          else acc[v] += w * (-1.f - p.eps * exp_mufu(z)) * tk;
        }
      }
    if (!kBackward) {
#pragma unroll
      for (int v = 0; v < V; ++v) { p.loss_pos[n * S + s0 + v] = acc[v]; lsum += acc[v]; }
    } else {
      float g[V];
#pragma unroll
      for (int v = 0; v < V; ++v) g[v] = grad_scale(p.gout, p.reduction, nullptr, (long long)p.N * S).at(n * S + s0 + v);
#pragma unroll
      for (int k = 0; k < KMAX; ++k)
        if (k < K) {
          const bool valid = !(ign && k == p.ignore_index);
          const float w = p.weight ? p.weight[k] : 1.f;
          Vec8<T> o;
#pragma unroll
          for (int v = 0; v < V; ++v) {
            const float lp = to_f(r[k].v[v]) - lse[v];
            float ck = 0.f;
            if (valid) {
              const float tk = to_f(q[k].v[v]);
              ck = w * (-1.f - p.eps * exp_mufu(lp * tk)) * tk;
            }
            o.v[v] = from_f<T>(g[v] * (ck - exp_mufu(lp) * acc[v]));
          }
          st8(dx + off + (size_t)k * S, o);
        }
    }
  }
  if (!kBackward) store_partials(p.partials, red, lsum, V * thread_iters(pv0, PV, stride));
}

template <typename T>
bool vec_eligible(const LossParams& p) {
  constexpr int V = Vec8<T>::N;
  auto al8 = [](const void* q) { return q == nullptr || (reinterpret_cast<uintptr_t>(q) & 7) == 0; };
  return p.S > 1 && p.S % V == 0 && p.K <= 32 && (long long)p.K * p.S < 0x7fffffffLL && al8(p.x) && al8(p.soft) && al8(p.dx);
}

// ---- host dispatch ---------------------------------------------------------------------------------
// f(std::integral_constant<int, KMAX>{}) for the smallest register-column instantiation that holds K (K <= 32)
template <class F>
void dispatch_kmax(int K, F f) {
  switch ((K + 3) / 4) {
    case 0: case 1: f(std::integral_constant<int, 4>{}); break;
    case 2: f(std::integral_constant<int, 8>{}); break;
    case 3: f(std::integral_constant<int, 12>{}); break;
    case 4: f(std::integral_constant<int, 16>{}); break;
    case 5: f(std::integral_constant<int, 20>{}); break;
    case 6: f(std::integral_constant<int, 24>{}); break;
    case 7: f(std::integral_constant<int, 28>{}); break;
    default: f(std::integral_constant<int, 32>{}); break;
  }
}

// The focal / poly-1 entry points: the register-column kernel when it applies, else the scalar kernel (hard targets: a
// warp per position at S == 1; soft targets: a thread per position); the forward then folds the partials into fwd_out.
template <bool kSoft, bool kBackward>
int class_loss(const LossParams& p, float* fwd_out, int dtype, void* stream) {
  const long long P = (long long)p.N * p.S;
  if (P == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  int grid = 0;
  const int rc = dispatch_dtype(dtype, [&](auto type) {
    using T = typename decltype(type)::type;
    if (vec_eligible<T>(p)) {
      grid = grid_for(P / Vec8<T>::N, kThreads);
      dispatch_kmax(p.K, [&](auto kmax) {
        constexpr int KMAX = decltype(kmax)::value;
        if constexpr (kSoft) poly_soft_vec_kernel<T, KMAX, kBackward><<<grid, kThreads, 0, st>>>(p);
        else hard_vec_kernel<T, KMAX, kBackward><<<grid, kThreads, 0, st>>>(p);
      });
    } else if constexpr (kSoft) {
      grid = grid_for(P, kThreads);
      poly_soft_kernel<T, kBackward><<<grid, kThreads, 0, st>>>(p);
    } else {
      grid = grid_for(P, p.S == 1 ? kThreads / 32 : kThreads);
      hard_kernel<T, kBackward><<<grid, kThreads, 0, st>>>(p);
    }
    HB_LAUNCH_CHECK();
    return 0;
  });
  if (rc != 0 || kBackward) return rc;
  finalize_kernel<2><<<1, 32, 0, st>>>(p.partials, grid, (double)P, 0.f, fwd_out);
  HB_LAUNCH_CHECK();
  return 0;
}

// ---- dice -----------------------------------------------------------------------------------------
// part[(k * gridDim.x + bx) * 2 + {0, 1}] = this block's {sum x*t, sum (x + gamma*t)} of class k; grid = (blocks per class, K).
// Per-block partials combined in a fixed order by dice_finalize_kernel: deterministic (the first version atomically added
// doubles). (n, k) planes are contiguous runs of S elements: 128-bit loads when S is a multiple of the vector width.
template <typename T>
__global__ void __launch_bounds__(kThreads) dice_sums_kernel(const T* __restrict__ x, const T* __restrict__ t, int N, int K,
                                                             long long S, float gamma, double* part, int vec) {
  constexpr int V = Vec16<T>::N;
  __shared__ double red[32];
  const int k = blockIdx.y;
  double a = 0.0, c = 0.0;
  float fa = 0.f, fc = 0.f;
  const long long stride = (long long)gridDim.x * kThreads;
  int cnt = 0;
  if (vec) {
    const long long SV = S / V, total = (long long)N * SV;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += stride) {
      const long long n = i / SV, sv = i - n * SV;
      const long long off = (n * K + k) * S + sv * V;
      const Vec16<T> xv = ld16_stream(x + off), tv = ld16_stream(t + off);
#pragma unroll
      for (int j = 0; j < V; ++j) {
        const float xf = to_f(xv.v[j]), tf = to_f(tv.v[j]);
        fa = fmaf(xf, tf, fa);
        fc += xf + gamma * tf;
      }
      if (++cnt == 32) { a += fa; c += fc; fa = fc = 0.f; cnt = 0; }  // bounded fp32 partials
    }
  } else {
    const long long per_class = (long long)N * S;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < per_class; i += stride) {
      const long long n = i / S, s = i % S;
      const long long off = (n * K + k) * S + s;
      const float xv = to_f(x[off]), tv = to_f(t[off]);
      fa = fmaf(xv, tv, fa);
      fc += xv + gamma * tv;
      if (++cnt == 256) { a += fa; c += fc; fa = fc = 0.f; cnt = 0; }
    }
  }
  a += fa; c += fc;
  a = block_sum<double>(a, red);
  c = block_sum<double>(c, red);
  if (threadIdx.x == 0) {
    part[((size_t)k * gridDim.x + blockIdx.x) * 2] = a;
    part[((size_t)k * gridDim.x + blockIdx.x) * 2 + 1] = c;
  }
}

// loss = 1 - (1 + 1/gamma) * sum_k w_k * dice_k / sum_k w_k,  dice_k = (gamma*I_k + eps) / (C_k + eps)
// also emits coef[k] = {d loss / d I_k', d loss / d C_k} pieces used by the backward: for element (k):
//   dloss/dx = -(1+1/gamma) * wn_k * (gamma * t * (C_k+eps) - (gamma*I_k+eps)) / (C_k+eps)^2
// One block: warp w folds the gx partials of classes w, w + 8, ... (lanes stride, shuffle tree), then thread 0 combines.
__global__ void __launch_bounds__(kThreads) dice_finalize_kernel(const double* part, int gx, double* sums, const float* weight,
                                                                 int K, float gamma, float eps, float* out,
                                                                 float* coef /*[K][2]*/) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k = warp; k < K; k += kThreads / 32) {
    double a = 0.0, c = 0.0;
    for (int i = lane; i < gx; i += 32) { a += part[((size_t)k * gx + i) * 2]; c += part[((size_t)k * gx + i) * 2 + 1]; }
    a = warp_sum(a);
    c = warp_sum(c);
    if (lane == 0) { sums[2 * k] = a; sums[2 * k + 1] = c; }
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double wsum = 0.0, acc = 0.0;
  for (int k = 0; k < K; ++k) {
    const double w = weight ? (double)weight[k] : 1.0;
    const double inter = (double)gamma * sums[2 * k] + (double)eps;
    const double card = sums[2 * k + 1] + (double)eps;
    acc += w * inter / card;
    wsum += w;
  }
  const double f = 1.0 + 1.0 / (double)gamma;
  out[0] = (float)(1.0 - f * acc / wsum);
  for (int k = 0; k < K; ++k) {
    const double w = (weight ? (double)weight[k] : 1.0) / wsum;
    const double inter = (double)gamma * sums[2 * k] + (double)eps;
    const double card = sums[2 * k + 1] + (double)eps;
    coef[2 * k] = (float)(-f * w * (double)gamma / card);       // multiplies t
    coef[2 * k + 1] = (float)(f * w * inter / (card * card));   // constant term
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) dice_bwd_kernel(const T* __restrict__ t, const float* __restrict__ coef,
                                                            const float* __restrict__ gout, T* __restrict__ dx, int N,
                                                            int K, long long S, int vec) {
  constexpr int V = Vec16<T>::N;
  const long long stride = (long long)gridDim.x * kThreads;
  const float g = gout[0];
  if (vec) {
    const long long SV = S / V, total = (long long)N * K * SV;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += stride) {
      const int k = (int)((i / SV) % K);
      const float c0 = g * coef[2 * k], c1 = g * coef[2 * k + 1];
      const Vec16<T> tv = ld16_stream(t + i * V);
      Vec16<T> o;
#pragma unroll
      for (int j = 0; j < V; ++j) o.v[j] = from_f<T>(fmaf(c0, to_f(tv.v[j]), c1));
      st16(dx + i * V, o);
    }
    return;
  }
  const long long total = (long long)N * K * S;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += stride) {
    const int k = (int)((i / S) % K);
    dx[i] = from_f<T>(g * fmaf(coef[2 * k], to_f(t[i]), coef[2 * k + 1]));
  }
}

int dice_blocks_per_class(long long per_class, int K) {
  int gx = grid_for(per_class, kThreads * 16);
  if ((long long)gx * K > HB_NUM_SMS * 16) gx = (HB_NUM_SMS * 16 + K - 1) / K;
  return gx < 1 ? 1 : gx;
}

// ---- complement cross entropy ---------------------------------------------------------------------
// per position (target y, A = the classes k != y outside the ignored column):
//   L = w_y * ce * [y != ignore_index] + gamma * C,   ce = lse - x_y,
//   C = -1/(K-1) * sum_{k in A} w_k q_k log q_k,    log q_k = x_k - lse_{k != y}
// (q is the softmax over the non-target classes - the reference's p_k / (1 - p_y) without the cancellation of 1 - p_y).
//   dC/dx_y = 0,   dC/dx_j = -1/(K-1) * q_j * ([j in A] w_j (1 + log q_j) - sum_{k in A} w_k q_k (1 + log q_k))
// The CE part follows torch: any ignore_index value drops the row. The complement term drops the ignored column only.
// partials[3 * block + {0, 1, 2}] = {sum of w_y * ce over the non-ignored positions, sum of their w_y, sum of C}.
template <typename T, bool kBackward, class Ln>
__device__ __forceinline__ void cce_position(const LossParams& p, const Ln& ln, const T* xp, T* dp, long long st,
                                             long long pos, double& sa, double& sb, double& sc) {
  const int K = p.K;
  auto x_at = [&](int k) { return to_f(xp[k * st]); };
  auto w_at = [&](int k) { return p.weight ? p.weight[k] : 1.f; };
  const long long tl = p.target[pos];
  const bool inr = tl >= 0 && tl < K;
  const int t = inr ? (int)tl : -1;
  const bool comp = p.gamma != 0.f;
  const int icol = (p.ignore_index >= 0 && p.ignore_index < K) ? p.ignore_index : -1;
  float mx = -INFINITY, mc = -INFINITY;
  for (int k = ln.k0; k < K; k += Ln::kStep) {
    const float v = x_at(k);
    mx = fmaxf(mx, v);
    if (k != t) mc = fmaxf(mc, v);
  }
  mx = ln.max(mx);
  mc = ln.max(mc);
  float s = 0.f, sn = 0.f;
  for (int k = ln.k0; k < K; k += Ln::kStep) {
    const float v = x_at(k);
    s += expf(v - mx);
    if (comp && k != t) sn += expf(v - mc);
  }
  s = ln.sum(s);
  sn = ln.sum(sn);
  const float lse = mx + logf(s), lsen = mc + logf(sn);
  // forward: sum_{k in A} w_k q_k log q_k; backward: sum_{k in A} w_k q_k (1 + log q_k)
  float acc = 0.f;
  if (comp && inr) {
    for (int k = ln.k0; k < K; k += Ln::kStep)
      if (k != t && k != icol) {
        const float lq = x_at(k) - lsen;
        acc += w_at(k) * expf(lq) * (kBackward ? 1.f + lq : lq);
      }
    acc = ln.sum(acc);
  }
  const float inv = 1.f / (float)(K - 1);
  if (!kBackward) {
    float wce = 0.f, wv = 0.f;
    if (tl != p.ignore_index) {
      if (inr) { wv = w_at(t); wce = wv * (lse - x_at(t)); } else { wce = NAN; }
    }
    const float c = comp ? (inr ? -inv * acc : NAN) : 0.f;
    if (ln.k0 == 0) {
      p.loss_pos[pos] = wce + p.gamma * c;
      sa += wce; sb += wv; sc += c;
    }
  } else {
    const long long P = (long long)p.N * p.S;
    const float gce = grad_scale(p.gout, p.reduction, p.fwd_out + 1, P).at(pos);
    const float gc = grad_scale(p.gout, p.reduction, nullptr, P).at(pos);
    const float cw = (inr && tl != p.ignore_index) ? gce * w_at(t) : 0.f;
    const float cc = (comp && inr) ? -p.gamma * gc * inv : 0.f;
    for (int k = ln.k0; k < K; k += Ln::kStep) {
      const float v = x_at(k);
      float d = cw * (expf(v - lse) - (k == t ? 1.f : 0.f));
      if (comp && inr && k != t) {  // lsen is -inf without the complement term
        const float lq = v - lsen;
        d += cc * expf(lq) * ((k != icol ? w_at(k) * (1.f + lq) : 0.f) - acc);
      }
      dp[k * st] = from_f<T>(d);
    }
  }
}

template <typename T, bool kBackward>
__global__ void __launch_bounds__(kThreads) cce_kernel(LossParams p) {
  __shared__ double red[32];
  double sa = 0.0, sb = 0.0, sc = 0.0;
  for_each_position<T>(p, [&](const auto& ln, const T* xp, T* dp, long long st, long long pos) {
    cce_position<T, kBackward>(p, ln, xp, dp, st, pos, sa, sb, sc);
  });
  if (!kBackward) store_partials(p.partials, red, sa, sb, sc);
}

// ---- mutual channel loss --------------------------------------------------------------------------
// x is [N, C = cnum * xi, S]; row r = n * C + ch (one channel of one sample) is a contiguous run of S values.
//   discriminative part: d_c = max_j (x[c*xi + j] * mask[c][j]) (masked channels enter as 0 * x), torch cross entropy of
//     d over the cnum classes;
//   diversity part: per position, the mean over classes of max_j softmax_s(x[c*xi + j])  (softmax over the spatial axis);
//   L = discr - alpha * diversity.
// Argmaxes take the first index on ties, as the CPU max does.
struct McParams {
  const void* x;
  const long long* target;      // [N, S]
  const float* weight;          // [cnum] or null
  const unsigned char* mask;    // [cnum * xi]
  const float* row_lse;         // [N * C]: log sum_s exp(x) of every row (pass A)
  float* loss_pos;              // [N * S]
  float* lse_d;                 // [N * S]: log-sum-exp of d over the classes (saved for the backward)
  double* partials;             // [grid][3]
  const float* gout;
  const float* fwd_out;
  float* rdot;                  // [N * C]: sum_s G_s p_s of every row (pass C)
  void* dx;
  int N, cnum, xi, S, ignore_index, reduction;
  float alpha;
};

// pass A: one block per row, online (max, sum exp) merged across the block in a fixed order
__device__ __forceinline__ void lse_merge(float& m, float& z, float m2, float z2) {
  const float mn = fmaxf(m, m2);
  if (mn == -INFINITY) return;
  z = z * expf(m - mn) + z2 * expf(m2 - mn);
  m = mn;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) mcl_row_lse_kernel(const T* __restrict__ x, long long S, int vec, float* row_lse) {
  constexpr int V = Vec16<T>::N;
  __shared__ float sm[32], sz[32];
  const T* row = x + (long long)blockIdx.x * S;
  float m = -INFINITY, z = 0.f;
  if (vec) {
    for (long long i = threadIdx.x; i < S / V; i += kThreads) {
      const Vec16<T> v = ld16_stream(row + i * V);
      float vm = -INFINITY;
#pragma unroll
      for (int j = 0; j < V; ++j) vm = fmaxf(vm, to_f(v.v[j]));
      float vz = 0.f;
#pragma unroll
      for (int j = 0; j < V; ++j) vz += expf(to_f(v.v[j]) - vm);
      lse_merge(m, z, vm, vz);
    }
  } else {
    for (long long i = threadIdx.x; i < S; i += kThreads) lse_merge(m, z, to_f(row[i]), 1.f);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), z2 = __shfl_xor_sync(0xffffffffu, z, o);
    lse_merge(m, z, m2, z2);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { sm[warp] = m; sz[warp] = z; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kThreads / 32; ++w) lse_merge(m, z, sm[w], sz[w]);
    row_lse[blockIdx.x] = m + logf(z);
  }
}

// class c at one position: the masked max (value, channel) and the largest spatial-softmax probability (value, channel)
template <typename T>
__device__ __forceinline__ void mcl_class(const McParams& p, const T* xc, const float* lse_c, const unsigned char* mc,
                                          float& d, int& jd, float& pv, int& jv) {
  for (int j = 0; j < p.xi; ++j) {
    const float v = to_f(xc[(long long)j * p.S]);
    const float dv = v * (float)mc[j];
    if (j == 0 || dv > d) { d = dv; jd = j; }
    const float pr = expf(v - lse_c[j]);
    if (j == 0 || pr > pv) { pv = pr; jv = j; }
  }
}

// pass B: one thread per position
template <typename T>
__global__ void __launch_bounds__(kThreads) mcl_fwd_kernel(McParams p) {
  __shared__ double red[32];
  const T* x = (const T*)p.x;
  const int C = p.cnum * p.xi;
  const long long P = (long long)p.N * p.S;
  double sa = 0.0, sb = 0.0, sc = 0.0;
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long pos = (long long)blockIdx.x * kThreads + threadIdx.x; pos < P; pos += stride) {
    const long long n = pos / p.S, s = pos % p.S;
    const T* xp = x + n * C * p.S + s;
    const float* lse_n = p.row_lse + n * C;
    const long long tl = p.target[pos];
    float m = -INFINITY, z = 0.f, dt = NAN, div = 0.f;
    for (int c = 0; c < p.cnum; ++c) {
      float d, pv;
      int jd, jv;
      mcl_class<T>(p, xp + (long long)c * p.xi * p.S, lse_n + c * p.xi, p.mask + c * p.xi, d, jd, pv, jv);
      lse_merge(m, z, d, 1.f);
      if (c == tl) dt = d;
      div += pv;
    }
    const float lse = m + logf(z);
    float wce = 0.f, wv = 0.f;
    if (tl != p.ignore_index) {
      if (tl >= 0 && tl < p.cnum) { wv = p.weight ? p.weight[tl] : 1.f; wce = wv * (lse - dt); } else { wce = NAN; }
    }
    div /= (float)p.cnum;
    p.loss_pos[pos] = wce - p.alpha * div;
    p.lse_d[pos] = lse;
    sa += wce; sb += wv; sc += div;
  }
  store_partials(p.partials, red, sa, sb, sc);
}

// pass C: one block per (sample, class); per row of the class R = sum_s G_s p_s with G_s = -(alpha/cnum) g_s at the
// positions where the row holds the class' largest probability. Per-thread, per-row sums live in shared memory.
template <typename T>
__global__ void __launch_bounds__(kThreads) mcl_rdot_kernel(McParams p) {
  extern __shared__ float acc[];  // [xi][blockDim.x]
  __shared__ double red[32];
  const int n = blockIdx.x / p.cnum, c = blockIdx.x % p.cnum;
  const int C = p.cnum * p.xi;
  const long long P = (long long)p.N * p.S;
  const T* xc = (const T*)p.x + ((long long)n * C + (long long)c * p.xi) * p.S;
  const float* lse_c = p.row_lse + (long long)n * C + c * p.xi;
  for (int j = 0; j < p.xi; ++j) acc[j * blockDim.x + threadIdx.x] = 0.f;
  for (long long s = threadIdx.x; s < p.S; s += blockDim.x) {
    const float g = grad_scale(p.gout, p.reduction, nullptr, P).at(n * p.S + s);
    float pv = 0.f;
    int jv = 0;
    for (int j = 0; j < p.xi; ++j) {
      const float pr = expf(to_f(xc[(long long)j * p.S + s]) - lse_c[j]);
      if (j == 0 || pr > pv) { pv = pr; jv = j; }
    }
    acc[jv * blockDim.x + threadIdx.x] += g * pv;
  }
  const float f = -p.alpha / (float)p.cnum;
  for (int j = 0; j < p.xi; ++j) {
    const double r = block_sum<double>((double)acc[j * blockDim.x + threadIdx.x], red);
    if (threadIdx.x == 0) p.rdot[(long long)n * C + c * p.xi + j] = f * (float)r;
  }
}

// pass D: one thread per position; dx = (CE gradient of d_c on its kept argmax channel) + p (G - R)
template <typename T>
__global__ void __launch_bounds__(kThreads) mcl_bwd_kernel(McParams p) {
  const T* x = (const T*)p.x;
  T* dx = (T*)p.dx;
  const int C = p.cnum * p.xi;
  const long long P = (long long)p.N * p.S;
  const float f = -p.alpha / (float)p.cnum;
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long pos = (long long)blockIdx.x * kThreads + threadIdx.x; pos < P; pos += stride) {
    const long long n = pos / p.S, s = pos % p.S;
    const long long off = n * C * p.S + s;
    const float* lse_n = p.row_lse + n * C;
    const float* rdot_n = p.rdot + n * C;
    const long long tl = p.target[pos];
    const float gdiv = grad_scale(p.gout, p.reduction, nullptr, P).at(pos);
    const bool ce_on = tl != p.ignore_index && tl >= 0 && tl < p.cnum;
    const float gce = ce_on ? grad_scale(p.gout, p.reduction, p.fwd_out + 1, P).at(pos) * (p.weight ? p.weight[tl] : 1.f)
                            : 0.f;
    const float lse = p.lse_d[pos];
    for (int c = 0; c < p.cnum; ++c) {
      const long long oc = off + (long long)c * p.xi * p.S;
      float d, pv;
      int jd, jv;
      mcl_class<T>(p, x + oc, lse_n + c * p.xi, p.mask + c * p.xi, d, jd, pv, jv);
      const float dd = gce * (expf(d - lse) - (c == tl ? 1.f : 0.f));
      for (int j = 0; j < p.xi; ++j) {
        const int ch = c * p.xi + j;
        const float pr = expf(to_f(x[oc + (long long)j * p.S]) - lse_n[ch]);
        float o = pr * ((j == jv ? f * gdiv : 0.f) - rdot_n[ch]);
        if (j == jd) o += dd * (float)p.mask[ch];
        dx[oc + (long long)j * p.S] = from_f<T>(o);
      }
    }
  }
}

// pass C block size: xi per-thread sums (plus the reduction scratch) must fit the default 48 KB of shared memory
int mcl_rdot_threads(int xi) {
  int t = (47 * 1024 / (int)sizeof(float) / xi) / 32 * 32;
  return t > kThreads ? kThreads : t;
}

// The shape checks of the entry points, before any launch or device query. N = 0 is an empty batch (nothing to do);
// K < 1 or S < 1 describe no class or no position of a non-empty tensor.
bool bad_nks(int N, int K, long long S) { return N < 0 || K < 1 || S < 1; }
// mcl_rdot_threads(xi) >= 32 for xi <= 376
bool bad_mcl(int N, int cnum, int xi, int S) { return bad_nks(N, cnum, S) || xi < 1 || mcl_rdot_threads(xi) < 32; }

}  // namespace

extern "C" {

// Upper bound of the number of partial-sum pairs a forward launch writes (size `partials` as 2*this doubles).
int hb_loss_max_partials(void) { return HB_NUM_SMS * 8; }

// kind: 0 focal, 1 poly. fwd_out: float[3] = {sum, valid count, mean}. loss_pos: float[N*S].
int hb_cls_loss_hard_fwd(const void* x, const long long* target, const float* weight, float* loss_pos, double* partials,
                         float* fwd_out, int N, int K, int S, int ignore_index, int kind, float gamma, float eps,
                         int dtype, void* stream) {
  if (bad_nks(N, K, S)) return (int)cudaErrorInvalidValue;
  LossParams p{};
  p.x = x; p.target = target; p.weight = weight; p.loss_pos = loss_pos; p.partials = partials;
  p.N = N; p.K = K; p.S = S; p.ignore_index = ignore_index; p.kind = kind; p.gamma = gamma; p.eps = eps;
  return class_loss<false, false>(p, fwd_out, dtype, stream);
}

// reduction: 0 none (gout[N*S]), 1 mean, 2 sum (gout[1]). dx has the dtype/shape of x.
int hb_cls_loss_hard_bwd(const void* x, const long long* target, const float* weight, const float* gout,
                         const float* fwd_out, void* dx, int N, int K, int S, int ignore_index, int kind, float gamma,
                         float eps, int reduction, int dtype, void* stream) {
  if (bad_nks(N, K, S)) return (int)cudaErrorInvalidValue;
  LossParams p{};
  p.x = x; p.target = target; p.weight = weight; p.gout = gout; p.fwd_out = fwd_out; p.dx = dx;
  p.N = N; p.K = K; p.S = S; p.ignore_index = ignore_index; p.kind = kind; p.reduction = reduction; p.gamma = gamma;
  p.eps = eps;
  return class_loss<false, true>(p, nullptr, dtype, stream);
}

int hb_poly_soft_fwd(const void* x, const void* soft, const float* weight, float* loss_pos, double* partials,
                     float* fwd_out, int N, int K, int S, int ignore_index, float eps, int dtype, void* stream) {
  if (bad_nks(N, K, S)) return (int)cudaErrorInvalidValue;
  LossParams p{};
  p.x = x; p.soft = soft; p.weight = weight; p.loss_pos = loss_pos; p.partials = partials;
  p.N = N; p.K = K; p.S = S; p.ignore_index = ignore_index; p.kind = POLY; p.eps = eps;
  return class_loss<true, false>(p, fwd_out, dtype, stream);
}

int hb_poly_soft_bwd(const void* x, const void* soft, const float* weight, const float* gout, void* dx, int N, int K,
                     int S, int ignore_index, float eps, int reduction, int dtype, void* stream) {
  if (bad_nks(N, K, S)) return (int)cudaErrorInvalidValue;
  LossParams p{};
  p.x = x; p.soft = soft; p.weight = weight; p.gout = gout; p.dx = dx;
  p.N = N; p.K = K; p.S = S; p.ignore_index = ignore_index; p.kind = POLY; p.reduction = reduction; p.eps = eps;
  return class_loss<true, true>(p, nullptr, dtype, stream);
}

// scratch: double[hb_dice_scratch_doubles(K)] (per-block partials + the K folded pairs); out: float[1]; coef: float[2K]
size_t hb_dice_scratch_doubles(int K) { return 2 * ((size_t)HB_NUM_SMS * 16 + (size_t)K) + 2 * (size_t)K; }

int hb_dice_fwd(const void* x, const void* target, const float* weight, double* scratch, float* out, float* coef, int N,
                int K, long long S, float gamma, float eps, int dtype, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (bad_nks(N, K, S) || K > 65535) return (int)cudaErrorInvalidValue;
  const int gx = dice_blocks_per_class((long long)N * S, K);
  double* part = scratch;
  double* sums = scratch + 2 * (size_t)gx * K;
  dim3 grid(gx, K);
  return dispatch_dtype(dtype, [&](auto type) {
    using T = typename decltype(type)::type;
    const int vec = S % Vec16<T>::N == 0 && aligned16(x) && aligned16(target);
    dice_sums_kernel<T><<<grid, kThreads, 0, st>>>((const T*)x, (const T*)target, N, K, S, gamma, part, vec);
    HB_LAUNCH_CHECK();
    dice_finalize_kernel<<<1, kThreads, 0, st>>>(part, gx, sums, weight, K, gamma, eps, out, coef);
    HB_LAUNCH_CHECK();
    return 0;
  });
}

int hb_dice_bwd(const void* target, const float* coef, const float* gout, void* dx, int N, int K, long long S, int dtype,
                void* stream) {
  if (bad_nks(N, K, S)) return (int)cudaErrorInvalidValue;
  const long long total = (long long)N * K * S;
  if (total == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_dtype(dtype, [&](auto type) {
    using T = typename decltype(type)::type;
    const int vec = S % Vec16<T>::N == 0 && aligned16(target) && aligned16(dx);
    const int grid = grid_for(total, kThreads * (vec ? Vec16<T>::N * 2 : 4));
    dice_bwd_kernel<T><<<grid, kThreads, 0, st>>>((const T*)target, coef, gout, (T*)dx, N, K, S, vec);
    HB_LAUNCH_CHECK();
    return 0;
  });
}

int hb_cce_fwd(const void* x, const long long* target, const float* weight, float* loss_pos, double* partials,
               float* fwd_out, int N, int K, int S, int ignore_index, float gamma, int dtype, void* stream) {
  if (bad_nks(N, K, S) || (gamma != 0.f && K < 2)) return (int)cudaErrorInvalidValue;  // C divides by K - 1
  LossParams p{};
  p.x = x; p.target = target; p.weight = weight; p.loss_pos = loss_pos; p.partials = partials;
  p.N = N; p.K = K; p.S = S; p.ignore_index = ignore_index; p.gamma = gamma;
  const long long P = (long long)N * S;
  if (P == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = grid_for(P, S == 1 ? kThreads / 32 : kThreads);
  return dispatch_dtype(dtype, [&](auto type) {
    using T = typename decltype(type)::type;
    cce_kernel<T, false><<<grid, kThreads, 0, st>>>(p);
    HB_LAUNCH_CHECK();
    finalize_kernel<3><<<1, 32, 0, st>>>(partials, grid, (double)P, gamma, fwd_out);
    HB_LAUNCH_CHECK();
    return 0;
  });
}

int hb_cce_bwd(const void* x, const long long* target, const float* weight, const float* gout, const float* fwd_out,
               void* dx, int N, int K, int S, int ignore_index, float gamma, int reduction, int dtype, void* stream) {
  if (bad_nks(N, K, S) || (gamma != 0.f && K < 2)) return (int)cudaErrorInvalidValue;  // C divides by K - 1
  LossParams p{};
  p.x = x; p.target = target; p.weight = weight; p.gout = gout; p.fwd_out = fwd_out; p.dx = dx;
  p.N = N; p.K = K; p.S = S; p.ignore_index = ignore_index; p.reduction = reduction; p.gamma = gamma;
  const long long P = (long long)N * S;
  if (P == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = grid_for(P, S == 1 ? kThreads / 32 : kThreads);
  return dispatch_dtype(dtype, [&](auto type) {
    cce_kernel<typename decltype(type)::type, true><<<grid, kThreads, 0, st>>>(p);
    HB_LAUNCH_CHECK();
    return 0;
  });
}

int hb_mcl_fwd(const void* x, const long long* target, const float* weight, const unsigned char* mask, float* row_lse,
               float* loss_pos, float* lse_d, double* partials, float* fwd_out, int N, int cnum, int xi, int S,
               int ignore_index, float alpha, int dtype, void* stream) {
  if (bad_mcl(N, cnum, xi, S)) return (int)cudaErrorInvalidValue;
  McParams p{};
  p.x = x; p.target = target; p.weight = weight; p.mask = mask; p.row_lse = row_lse; p.loss_pos = loss_pos;
  p.lse_d = lse_d; p.partials = partials;
  p.N = N; p.cnum = cnum; p.xi = xi; p.S = S; p.ignore_index = ignore_index; p.alpha = alpha;
  const long long P = (long long)N * S, rows = (long long)N * cnum * xi;
  if (P == 0 || rows == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = grid_for(P, kThreads);
  return dispatch_dtype(dtype, [&](auto type) {
    using T = typename decltype(type)::type;
    const int vec = S % Vec16<T>::N == 0 && aligned16(x);
    mcl_row_lse_kernel<T><<<(unsigned)rows, kThreads, 0, st>>>((const T*)x, S, vec, row_lse);
    HB_LAUNCH_CHECK();
    mcl_fwd_kernel<T><<<grid, kThreads, 0, st>>>(p);
    HB_LAUNCH_CHECK();
    finalize_kernel<3><<<1, 32, 0, st>>>(partials, grid, (double)P, -alpha, fwd_out);
    HB_LAUNCH_CHECK();
    return 0;
  });
}

int hb_mcl_bwd(const void* x, const long long* target, const float* weight, const unsigned char* mask,
               const float* row_lse, const float* lse_d, const float* gout, const float* fwd_out, float* rdot, void* dx,
               int N, int cnum, int xi, int S, int ignore_index, float alpha, int reduction, int dtype, void* stream) {
  if (bad_mcl(N, cnum, xi, S)) return (int)cudaErrorInvalidValue;
  McParams p{};
  p.x = x; p.target = target; p.weight = weight; p.mask = mask; p.row_lse = row_lse; p.lse_d = const_cast<float*>(lse_d); p.gout = gout;
  p.fwd_out = fwd_out; p.rdot = rdot; p.dx = dx;
  p.N = N; p.cnum = cnum; p.xi = xi; p.S = S; p.ignore_index = ignore_index; p.alpha = alpha; p.reduction = reduction;
  const long long P = (long long)N * S, groups = (long long)N * cnum;
  if (P == 0 || groups == 0) return 0;
  const int rt = mcl_rdot_threads(xi);
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = grid_for(P, kThreads);
  const size_t smem = (size_t)xi * rt * sizeof(float);
  return dispatch_dtype(dtype, [&](auto type) {
    using T = typename decltype(type)::type;
    mcl_rdot_kernel<T><<<(unsigned)groups, rt, smem, st>>>(p);
    HB_LAUNCH_CHECK();
    mcl_bwd_kernel<T><<<grid, kThreads, 0, st>>>(p);
    HB_LAUNCH_CHECK();
    return 0;
  });
}

}  // extern "C"
