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
#include "common.cuh"

namespace {

using namespace hb;

constexpr int kThreads = 256;

enum LossKind { FOCAL = 0, POLY = 1 };

struct LossParams {
  const void* x;            // [N, K, S]
  const long long* target;  // [N, S] hard targets (int64)         (hard)
  const void* soft;         // [N, K, S] soft targets, same dtype  (soft)
  const float* weight;      // [K] or null
  float* loss_pos;          // [N*S] per-position loss
  double* partials;         // [grid][2]: sum of valid losses, number of valid positions
  int N, K, S;
  int ignore_index;         // honoured only when 0 <= ignore_index < K (reference quirk)
  int kind;
  float gamma, eps;
};

template <typename T, typename Acc>
__device__ __forceinline__ float lse_thread(Acc x_at, int K) {
  float mx = -INFINITY;
  for (int k = 0; k < K; ++k) mx = fmaxf(mx, x_at(k));
  float s = 0.f;
  for (int k = 0; k < K; ++k) s += expf(x_at(k) - mx);
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

// ---- hard targets, forward ------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads) hard_fwd_kernel(LossParams p) {
  __shared__ double red[32];
  const T* x = (const T*)p.x;
  const long long P = (long long)p.N * p.S;
  double lsum = 0.0, lcnt = 0.0;
  const bool ign = p.ignore_index >= 0 && p.ignore_index < p.K;
  if (p.S == 1) {
    const int lane = threadIdx.x & 31;
    const long long warps = (long long)gridDim.x * (kThreads / 32);
    for (long long pos = (long long)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5); pos < P; pos += warps) {
      const T* row = x + pos * p.K;
      float mx = -INFINITY;
      for (int k = lane; k < p.K; k += 32) mx = fmaxf(mx, to_f(row[k]));
      mx = warp_max(mx);
      float s = 0.f;
      for (int k = lane; k < p.K; k += 32) s += expf(to_f(row[k]) - mx);
      s = warp_sum(s);
      if (lane == 0) {
        const long long t = p.target[pos];
        float l = NAN;
        if (t >= 0 && t < p.K) {
          const float logpt = to_f(row[t]) - (mx + logf(s));
          l = hard_loss(p, logpt, p.weight ? p.weight[t] : 1.f);
        }
        p.loss_pos[pos] = l;
        if (!(ign && t == p.ignore_index)) { lsum += l; lcnt += 1.0; }
      }
    }
  } else {
    const long long stride = (long long)gridDim.x * kThreads;
    for (long long pos = (long long)blockIdx.x * kThreads + threadIdx.x; pos < P; pos += stride) {
      const long long n = pos / p.S, s = pos % p.S;
      const T* base = x + n * p.K * p.S + s;
      auto x_at = [&](int k) { return to_f(base[(long long)k * p.S]); };
      const float lse = lse_thread<T>(x_at, p.K);
      const long long t = p.target[pos];
      float l = NAN;
      if (t >= 0 && t < p.K) l = hard_loss(p, x_at((int)t) - lse, p.weight ? p.weight[t] : 1.f);
      p.loss_pos[pos] = l;
      if (!(ign && t == p.ignore_index)) { lsum += l; lcnt += 1.0; }
    }
  }
  lsum = block_sum<double>(lsum, red);
  lcnt = block_sum<double>(lcnt, red);
  if (threadIdx.x == 0) { p.partials[2 * blockIdx.x] = lsum; p.partials[2 * blockIdx.x + 1] = lcnt; }
}

// out[0] = sum, out[1] = count, out[2] = mean  (fixed summation order)
__global__ void finalize_kernel(const double* partials, int n, float* out) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    double s = 0.0, c = 0.0;
    for (int i = 0; i < n; ++i) { s += partials[2 * i]; c += partials[2 * i + 1]; }
    out[0] = (float)s;
    out[1] = (float)c;
    out[2] = (float)(s / c);
  }
}

// ---- hard targets, backward -----------------------------------------------------------------------
struct LossBwdParams {
  LossParams f;
  const float* gout;    // reduction none: [N*S]; else 1 element
  const float* fwd_out; // {sum, count, mean} from the forward (count used for 'mean')
  void* dx;             // [N, K, S]
  int reduction;        // 0 none, 1 mean, 2 sum
};

template <typename T>
__global__ void __launch_bounds__(kThreads) hard_bwd_kernel(LossBwdParams b) {
  const LossParams& p = b.f;
  const T* x = (const T*)p.x;
  T* dx = (T*)b.dx;
  const long long P = (long long)p.N * p.S;
  const bool ign = p.ignore_index >= 0 && p.ignore_index < p.K;
  const float gscale = b.reduction == 1 ? b.gout[0] / b.fwd_out[1] : (b.reduction == 2 ? b.gout[0] : 0.f);
  if (p.S == 1) {
    const int lane = threadIdx.x & 31;
    const long long warps = (long long)gridDim.x * (kThreads / 32);
    for (long long pos = (long long)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5); pos < P; pos += warps) {
      const T* row = x + pos * p.K;
      float mx = -INFINITY;
      for (int k = lane; k < p.K; k += 32) mx = fmaxf(mx, to_f(row[k]));
      mx = warp_max(mx);
      float s = 0.f;
      for (int k = lane; k < p.K; k += 32) s += expf(to_f(row[k]) - mx);
      s = warp_sum(s);
      const float lse = mx + logf(s);
      const long long t = p.target[pos];
      float g = b.reduction == 0 ? b.gout[pos] : ((ign && t == p.ignore_index) ? 0.f : gscale);
      float c = 0.f;
      if (t >= 0 && t < p.K) c = g * hard_dloss(p, to_f(row[t]) - lse, p.weight ? p.weight[t] : 1.f);
      for (int k = lane; k < p.K; k += 32) {
        const float pk = expf(to_f(row[k]) - lse);
        dx[pos * p.K + k] = from_f<T>(c * ((k == t ? 1.f : 0.f) - pk));
      }
    }
  } else {
    const long long stride = (long long)gridDim.x * kThreads;
    for (long long pos = (long long)blockIdx.x * kThreads + threadIdx.x; pos < P; pos += stride) {
      const long long n = pos / p.S, s = pos % p.S;
      const long long off = n * p.K * p.S + s;
      auto x_at = [&](int k) { return to_f(x[off + (long long)k * p.S]); };
      const float lse = lse_thread<T>(x_at, p.K);
      const long long t = p.target[pos];
      float g = b.reduction == 0 ? b.gout[pos] : ((ign && t == p.ignore_index) ? 0.f : gscale);
      float c = 0.f;
      if (t >= 0 && t < p.K) c = g * hard_dloss(p, x_at((int)t) - lse, p.weight ? p.weight[t] : 1.f);
      for (int k = 0; k < p.K; ++k) {
        const float pk = expf(x_at(k) - lse);
        dx[off + (long long)k * p.S] = from_f<T>(c * ((k == t ? 1.f : 0.f) - pk));
      }
    }
  }
}

// ---- poly loss with soft targets ------------------------------------------------------------------
// per position: L = sum_{k valid} w_k * (-z_k + eps * (1 - exp(z_k))),  z_k = log_softmax(x)_k * t_k
template <typename T, bool kBackward>
__global__ void __launch_bounds__(kThreads) poly_soft_kernel(LossBwdParams b) {
  __shared__ double red[32];
  const LossParams& p = b.f;
  const T* x = (const T*)p.x;
  const T* tg = (const T*)p.soft;
  T* dx = (T*)b.dx;
  const long long P = (long long)p.N * p.S;
  const bool ign = p.ignore_index >= 0 && p.ignore_index < p.K;
  double lsum = 0.0;
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long pos = (long long)blockIdx.x * kThreads + threadIdx.x; pos < P; pos += stride) {
    const long long n = pos / p.S, s = pos % p.S;
    const long long off = n * p.K * p.S + s;
    auto x_at = [&](int k) { return to_f(x[off + (long long)k * p.S]); };
    const float lse = lse_thread<T>(x_at, p.K);
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
      const float g = b.reduction == 0 ? b.gout[pos] : (b.reduction == 1 ? b.gout[0] / (float)P : b.gout[0]);
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
  if (!kBackward) {
    lsum = block_sum<double>(lsum, red);
    if (threadIdx.x == 0) { p.partials[2 * blockIdx.x] = lsum; p.partials[2 * blockIdx.x + 1] = 0.0; }
  }
}

__global__ void finalize_soft_kernel(const double* partials, int n, double P, float* out) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < n; ++i) s += partials[2 * i];
    out[0] = (float)s;
    out[1] = (float)P;
    out[2] = (float)(s / P);
  }
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
template <typename T, int KMAX, bool kBackward>
__global__ void __launch_bounds__(kThreads) hard_vec_kernel(LossBwdParams b) {
  constexpr int V = Vec8<T>::N;
  __shared__ double red[32];
  const LossParams& p = b.f;
  const T* x = (const T*)p.x;
  T* dx = (T*)b.dx;
  const int K = p.K;
  const unsigned S = (unsigned)p.S, SV = S / V;
  const long long PV = (long long)p.N * SV;
  const bool ign = p.ignore_index >= 0 && p.ignore_index < K;
  float gscale = 0.f;
  if (kBackward) gscale = b.reduction == 1 ? b.gout[0] / b.fwd_out[1] : (b.reduction == 2 ? b.gout[0] : 0.f);
  double lsum = 0.0, lcnt = 0.0;
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long pv = (long long)blockIdx.x * kThreads + threadIdx.x; pv < PV; pv += stride) {
    const long long n = pv / SV;
    const unsigned s0 = (unsigned)(pv - n * SV) * V;
    const T* xp = x + n * K * S + s0;
    // classes k >= K hold -inf: the compute loops below run unpredicated over KMAX (exp(-inf) = 0, never the max or the
    // target); two dozen `k < K` predicates kept live across the body made ptxas shuffle them through P2R / R2P
    Vec8<T> r[KMAX];
    {
      const T* pk = xp;
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
          r[k] = ld8(pk);
        } else {
#pragma unroll
          for (int v = 0; v < V; ++v) r[k].v[v] = neg_inf<T>();
        }
        pk += S;
      }
    }
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
    for (int v = 0; v < V; ++v) { mx[v] = -INFINITY; sum[v] = 0.f; xt[v] = 0.f; }
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const float f = to_f(r[k].v[v]);
        mx[v] = fmaxf(mx[v], f);
        xt[v] = t[v] == k ? f : xt[v];
      }
    }
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
#pragma unroll
      for (int v = 0; v < V; ++v) sum[v] += exp_shift(to_f(r[k].v[v]), mx[v]);
    }
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
        const float g = b.reduction == 0 ? b.gout[n * S + s0 + v] : (skip[v] ? 0.f : gscale);
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
  if (!kBackward) {
    lsum = block_sum<double>(lsum, red);
    lcnt = block_sum<double>(lcnt, red);
    if (threadIdx.x == 0) { p.partials[2 * blockIdx.x] = lsum; p.partials[2 * blockIdx.x + 1] = lcnt; }
  }
}

// soft-target poly loss, same layout: logits AND soft targets in registers
template <typename T, int KMAX, bool kBackward>
__global__ void __launch_bounds__(kThreads) poly_soft_vec_kernel(LossBwdParams b) {
  constexpr int V = Vec8<T>::N;
  __shared__ double red[32];
  const LossParams& p = b.f;
  const T* x = (const T*)p.x;
  const T* tg = (const T*)p.soft;
  T* dx = (T*)b.dx;
  const int K = p.K;
  const unsigned S = (unsigned)p.S, SV = S / V;
  const long long PV = (long long)p.N * SV;
  const bool ign = p.ignore_index >= 0 && p.ignore_index < K;
  double lsum = 0.0;
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long pv = (long long)blockIdx.x * kThreads + threadIdx.x; pv < PV; pv += stride) {
    const long long n = pv / SV;
    const unsigned s0 = (unsigned)(pv - n * SV) * V;
    const long long off = n * K * S + s0;
    Vec8<T> r[KMAX], q[KMAX];   // k >= K: logits -inf, soft targets 0
    {
      const T* pk = x + off;
      const T* qk = tg + off;
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
          r[k] = ld8(pk);
          q[k] = ld8(qk);
        } else {
#pragma unroll
          for (int v = 0; v < V; ++v) { r[k].v[v] = neg_inf<T>(); q[k].v[v] = from_f<T>(0.f); }
        }
        pk += S;
        qk += S;
      }
    }
    float mx[V], sum[V], lse[V];
#pragma unroll
    for (int v = 0; v < V; ++v) { mx[v] = -INFINITY; sum[v] = 0.f; }
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
#pragma unroll
      for (int v = 0; v < V; ++v) mx[v] = fmaxf(mx[v], to_f(r[k].v[v]));
    }
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
#pragma unroll
      for (int v = 0; v < V; ++v) sum[v] += exp_shift(to_f(r[k].v[v]), mx[v]);
    }
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
      for (int v = 0; v < V; ++v)
        g[v] = b.reduction == 0 ? b.gout[n * S + s0 + v]
                                : (b.reduction == 1 ? b.gout[0] / (float)((long long)p.N * S) : b.gout[0]);
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
  if (!kBackward) {
    lsum = block_sum<double>(lsum, red);
    if (threadIdx.x == 0) { p.partials[2 * blockIdx.x] = lsum; p.partials[2 * blockIdx.x + 1] = 0.0; }
  }
}

template <typename T>
bool vec_eligible(const LossBwdParams& b) {
  constexpr int V = Vec8<T>::N;
  const LossParams& p = b.f;
  auto al8 = [](const void* q) { return q == nullptr || (reinterpret_cast<uintptr_t>(q) & 7) == 0; };
  return p.S > 1 && p.S % V == 0 && p.K <= 32 && (long long)p.K * p.S < 0x7fffffffLL && al8(p.x) && al8(p.soft) && al8(b.dx);
}

// launches the smallest KMAX instantiation that holds K; returns the grid size, 0 if not eligible
#define HB_KMAX_DISPATCH(KERNEL, T, BWD, b, grid, st)                                   \
  do {                                                                                  \
    switch (((b).f.K + 3) / 4) {                                                        \
      case 0: case 1: KERNEL<T, 4, BWD><<<grid, kThreads, 0, st>>>(b); break;           \
      case 2: KERNEL<T, 8, BWD><<<grid, kThreads, 0, st>>>(b); break;                   \
      case 3: KERNEL<T, 12, BWD><<<grid, kThreads, 0, st>>>(b); break;                  \
      case 4: KERNEL<T, 16, BWD><<<grid, kThreads, 0, st>>>(b); break;                  \
      case 5: KERNEL<T, 20, BWD><<<grid, kThreads, 0, st>>>(b); break;                  \
      case 6: KERNEL<T, 24, BWD><<<grid, kThreads, 0, st>>>(b); break;                  \
      case 7: KERNEL<T, 28, BWD><<<grid, kThreads, 0, st>>>(b); break;                  \
      default: KERNEL<T, 32, BWD><<<grid, kThreads, 0, st>>>(b); break;                 \
    }                                                                                   \
  } while (0)

template <typename T, bool kBackward>
int launch_hard_vec(const LossBwdParams& b, cudaStream_t st) {
  if (!vec_eligible<T>(b)) return 0;
  const int grid = grid_for((long long)b.f.N * b.f.S / Vec8<T>::N, kThreads);
  HB_KMAX_DISPATCH(hard_vec_kernel, T, kBackward, b, grid, st);
  return grid;
}
template <typename T, bool kBackward>
int launch_soft_vec(const LossBwdParams& b, cudaStream_t st) {
  if (!vec_eligible<T>(b)) return 0;
  const int grid = grid_for((long long)b.f.N * b.f.S / Vec8<T>::N, kThreads);
  HB_KMAX_DISPATCH(poly_soft_vec_kernel, T, kBackward, b, grid, st);
  return grid;
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

// ---- losses with three partial sums: complement CE and the mutual channel loss ----------------------
// partials[3 * block + {0, 1, 2}] = {sum of w_y * ce over the non-ignored positions, sum of their w_y, sum of the second
// term}; out = {A + coef * C, B, A / B + coef * C / P}: torch's weighted-mean cross entropy plus coef times the plain mean.
__global__ void finalize3_kernel(const double* partials, int n, double P, float coef, float* out) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    double a = 0.0, b = 0.0, c = 0.0;
    for (int i = 0; i < n; ++i) { a += partials[3 * i]; b += partials[3 * i + 1]; c += partials[3 * i + 2]; }
    out[0] = (float)(a + (double)coef * c);
    out[1] = (float)b;
    out[2] = (float)(a / b + (double)coef * c / P);
  }
}

__device__ __forceinline__ void store3(double* partials, double a, double b, double c, double* red) {
  a = block_sum<double>(a, red);
  b = block_sum<double>(b, red);
  c = block_sum<double>(c, red);
  if (threadIdx.x == 0) { partials[3 * blockIdx.x] = a; partials[3 * blockIdx.x + 1] = b; partials[3 * blockIdx.x + 2] = c; }
}

// {d loss / d (w_y ce), d loss / d (second term)} of one position for the reduction (mean: the first over sum w_y)
__device__ __forceinline__ void grad_scales(const float* gout, const float* fwd_out, int reduction, long long pos,
                                            long long P, float& gce, float& g2) {
  if (reduction == 0) { gce = g2 = gout[pos]; return; }
  gce = g2 = gout[0];
  if (reduction == 1) { gce /= fwd_out[1]; g2 /= (float)P; }
}

// ---- complement cross entropy ---------------------------------------------------------------------
// per position (target y, A = the classes k != y outside the ignored column):
//   L = w_y * ce * [y != ignore_index] + gamma * C,   ce = lse - x_y,
//   C = -1/(K-1) * sum_{k in A} w_k q_k log q_k,    log q_k = x_k - lse_{k != y}
// (q is the softmax over the non-target classes - the reference's p_k / (1 - p_y) without the cancellation of 1 - p_y).
//   dC/dx_y = 0,   dC/dx_j = -1/(K-1) * q_j * ([j in A] w_j (1 + log q_j) - sum_{k in A} w_k q_k (1 + log q_k))
// The CE part follows torch: any ignore_index value drops the row. The complement term drops the ignored column only.
struct CceParams {
  const void* x;            // [N, K, S]
  const long long* target;  // [N, S]
  const float* weight;      // [K] or null
  float* loss_pos;          // [N*S]
  double* partials;         // [grid][3]
  const float* gout;        // backward: [N*S] (none) or 1 element
  const float* fwd_out;     // backward: {sum, sum w_y, mean} of the forward
  void* dx;
  int N, K, S, ignore_index, reduction;
  float gamma;
};

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

template <typename T, bool kBackward, class Ln>
__device__ __forceinline__ void cce_position(const CceParams& p, const Ln& ln, const T* xp, T* dp, long long st,
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
    float gce, gc;
    grad_scales(p.gout, p.fwd_out, p.reduction, pos, (long long)p.N * p.S, gce, gc);
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
__global__ void __launch_bounds__(kThreads) cce_kernel(CceParams p) {
  __shared__ double red[32];
  const T* x = (const T*)p.x;
  T* dx = (T*)p.dx;
  const long long P = (long long)p.N * p.S;
  double sa = 0.0, sb = 0.0, sc = 0.0;
  if (p.S == 1) {
    const WarpLanes ln{threadIdx.x & 31};
    const long long warps = (long long)gridDim.x * (kThreads / 32);
    for (long long pos = (long long)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5); pos < P; pos += warps)
      cce_position<T, kBackward>(p, ln, x + pos * p.K, dx + pos * p.K, 1, pos, sa, sb, sc);
  } else {
    const ThreadLanes ln{};
    const long long stride = (long long)gridDim.x * kThreads;
    for (long long pos = (long long)blockIdx.x * kThreads + threadIdx.x; pos < P; pos += stride) {
      const long long off = (pos / p.S) * p.K * p.S + pos % p.S;
      cce_position<T, kBackward>(p, ln, x + off, dx + off, p.S, pos, sa, sb, sc);
    }
  }
  if (!kBackward) store3(p.partials, sa, sb, sc, red);
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
  store3(p.partials, sa, sb, sc, red);
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
    float gce, g;
    grad_scales(p.gout, p.fwd_out, p.reduction, n * p.S + s, P, gce, g);
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
    float gce, gdiv;
    grad_scales(p.gout, p.fwd_out, p.reduction, pos, P, gce, gdiv);
    const bool ce_on = tl != p.ignore_index && tl >= 0 && tl < p.cnum;
    gce = ce_on ? gce * (p.weight ? p.weight[tl] : 1.f) : 0.f;
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
  const long long P = (long long)N * S;
  if (P == 0) return 0;
  int grid = 0;
  cudaStream_t st = (cudaStream_t)stream;
  LossBwdParams vb{};
  vb.f = p;
  switch (dtype) {
    case HB_DTYPE_F32: grid = launch_hard_vec<float, false>(vb, st); break;
    case HB_DTYPE_BF16: grid = launch_hard_vec<__nv_bfloat16, false>(vb, st); break;
    case HB_DTYPE_F16: grid = launch_hard_vec<__half, false>(vb, st); break;
    default: return (int)cudaErrorInvalidValue;
  }
  if (grid == 0) {
    grid = grid_for(P, S == 1 ? kThreads / 32 : kThreads);
    switch (dtype) {
      case HB_DTYPE_F32: hard_fwd_kernel<float><<<grid, kThreads, 0, st>>>(p); break;
      case HB_DTYPE_BF16: hard_fwd_kernel<__nv_bfloat16><<<grid, kThreads, 0, st>>>(p); break;
      default: hard_fwd_kernel<__half><<<grid, kThreads, 0, st>>>(p); break;
    }
  }
  HB_LAUNCH_CHECK();
  finalize_kernel<<<1, 32, 0, st>>>(partials, grid, fwd_out);
  HB_LAUNCH_CHECK();
  return 0;
}

// reduction: 0 none (gout[N*S]), 1 mean, 2 sum (gout[1]). dx has the dtype/shape of x.
int hb_cls_loss_hard_bwd(const void* x, const long long* target, const float* weight, const float* gout,
                         const float* fwd_out, void* dx, int N, int K, int S, int ignore_index, int kind, float gamma,
                         float eps, int reduction, int dtype, void* stream) {
  if (bad_nks(N, K, S)) return (int)cudaErrorInvalidValue;
  LossBwdParams b{};
  b.f.x = x; b.f.target = target; b.f.weight = weight;
  b.f.N = N; b.f.K = K; b.f.S = S; b.f.ignore_index = ignore_index; b.f.kind = kind; b.f.gamma = gamma; b.f.eps = eps;
  b.gout = gout; b.fwd_out = fwd_out; b.dx = dx; b.reduction = reduction;
  const long long P = (long long)N * S;
  if (P == 0) return 0;
  int grid = 0;
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case HB_DTYPE_F32: grid = launch_hard_vec<float, true>(b, st); break;
    case HB_DTYPE_BF16: grid = launch_hard_vec<__nv_bfloat16, true>(b, st); break;
    case HB_DTYPE_F16: grid = launch_hard_vec<__half, true>(b, st); break;
    default: return (int)cudaErrorInvalidValue;
  }
  if (grid == 0) {
    grid = grid_for(P, S == 1 ? kThreads / 32 : kThreads);
    switch (dtype) {
      case HB_DTYPE_F32: hard_bwd_kernel<float><<<grid, kThreads, 0, st>>>(b); break;
      case HB_DTYPE_BF16: hard_bwd_kernel<__nv_bfloat16><<<grid, kThreads, 0, st>>>(b); break;
      default: hard_bwd_kernel<__half><<<grid, kThreads, 0, st>>>(b); break;
    }
  }
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_poly_soft_fwd(const void* x, const void* soft, const float* weight, float* loss_pos, double* partials,
                     float* fwd_out, int N, int K, int S, int ignore_index, float eps, int dtype, void* stream) {
  if (bad_nks(N, K, S)) return (int)cudaErrorInvalidValue;
  LossBwdParams b{};
  b.f.x = x; b.f.soft = soft; b.f.weight = weight; b.f.loss_pos = loss_pos; b.f.partials = partials;
  b.f.N = N; b.f.K = K; b.f.S = S; b.f.ignore_index = ignore_index; b.f.kind = POLY; b.f.eps = eps;
  const long long P = (long long)N * S;
  if (P == 0) return 0;
  int grid = 0;
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case HB_DTYPE_F32: grid = launch_soft_vec<float, false>(b, st); break;
    case HB_DTYPE_BF16: grid = launch_soft_vec<__nv_bfloat16, false>(b, st); break;
    case HB_DTYPE_F16: grid = launch_soft_vec<__half, false>(b, st); break;
    default: return (int)cudaErrorInvalidValue;
  }
  if (grid == 0) {
    grid = grid_for(P, kThreads);
    switch (dtype) {
      case HB_DTYPE_F32: poly_soft_kernel<float, false><<<grid, kThreads, 0, st>>>(b); break;
      case HB_DTYPE_BF16: poly_soft_kernel<__nv_bfloat16, false><<<grid, kThreads, 0, st>>>(b); break;
      default: poly_soft_kernel<__half, false><<<grid, kThreads, 0, st>>>(b); break;
    }
  }
  HB_LAUNCH_CHECK();
  finalize_soft_kernel<<<1, 32, 0, st>>>(partials, grid, (double)P, fwd_out);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_poly_soft_bwd(const void* x, const void* soft, const float* weight, const float* gout, void* dx, int N, int K,
                     int S, int ignore_index, float eps, int reduction, int dtype, void* stream) {
  if (bad_nks(N, K, S)) return (int)cudaErrorInvalidValue;
  LossBwdParams b{};
  b.f.x = x; b.f.soft = soft; b.f.weight = weight;
  b.f.N = N; b.f.K = K; b.f.S = S; b.f.ignore_index = ignore_index; b.f.kind = POLY; b.f.eps = eps;
  b.gout = gout; b.dx = dx; b.reduction = reduction;
  const long long P = (long long)N * S;
  if (P == 0) return 0;
  int grid = 0;
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case HB_DTYPE_F32: grid = launch_soft_vec<float, true>(b, st); break;
    case HB_DTYPE_BF16: grid = launch_soft_vec<__nv_bfloat16, true>(b, st); break;
    case HB_DTYPE_F16: grid = launch_soft_vec<__half, true>(b, st); break;
    default: return (int)cudaErrorInvalidValue;
  }
  if (grid == 0) {
    grid = grid_for(P, kThreads);
    switch (dtype) {
      case HB_DTYPE_F32: poly_soft_kernel<float, true><<<grid, kThreads, 0, st>>>(b); break;
      case HB_DTYPE_BF16: poly_soft_kernel<__nv_bfloat16, true><<<grid, kThreads, 0, st>>>(b); break;
      default: poly_soft_kernel<__half, true><<<grid, kThreads, 0, st>>>(b); break;
    }
  }
  HB_LAUNCH_CHECK();
  return 0;
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
  switch (dtype) {
#define HB_DICE_SUMS(T)                                                                                         \
  {                                                                                                             \
    const int vec = S % Vec16<T>::N == 0 && aligned16(x) && aligned16(target);                                 \
    dice_sums_kernel<T><<<grid, kThreads, 0, st>>>((const T*)x, (const T*)target, N, K, S, gamma, part, vec); \
  }
    case HB_DTYPE_F32: HB_DICE_SUMS(float) break;
    case HB_DTYPE_BF16: HB_DICE_SUMS(__nv_bfloat16) break;
    case HB_DTYPE_F16: HB_DICE_SUMS(__half) break;
#undef HB_DICE_SUMS
    default: return (int)cudaErrorInvalidValue;
  }
  HB_LAUNCH_CHECK();
  dice_finalize_kernel<<<1, kThreads, 0, st>>>(part, gx, sums, weight, K, gamma, eps, out, coef);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_dice_bwd(const void* target, const float* coef, const float* gout, void* dx, int N, int K, long long S, int dtype,
                void* stream) {
  if (bad_nks(N, K, S)) return (int)cudaErrorInvalidValue;
  const long long total = (long long)N * K * S;
  if (total == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
#define HB_DICE_BWD(T)                                                                                     \
  {                                                                                                        \
    const int vec = S % Vec16<T>::N == 0 && aligned16(target) && aligned16(dx);                           \
    const int grid = grid_for(total, kThreads * (vec ? Vec16<T>::N * 2 : 4));                             \
    dice_bwd_kernel<T><<<grid, kThreads, 0, st>>>((const T*)target, coef, gout, (T*)dx, N, K, S, vec);    \
  }
    case HB_DTYPE_F32: HB_DICE_BWD(float) break;
    case HB_DTYPE_BF16: HB_DICE_BWD(__nv_bfloat16) break;
    case HB_DTYPE_F16: HB_DICE_BWD(__half) break;
#undef HB_DICE_BWD
    default: return (int)cudaErrorInvalidValue;
  }
  HB_LAUNCH_CHECK();
  return 0;
}

#define HB_LOSS_DTYPE_SWITCH(dtype, LAUNCH)              \
  switch (dtype) {                                       \
    case HB_DTYPE_F32: LAUNCH(float); break;             \
    case HB_DTYPE_BF16: LAUNCH(__nv_bfloat16); break;    \
    case HB_DTYPE_F16: LAUNCH(__half); break;            \
    default: return (int)cudaErrorInvalidValue;          \
  }

int hb_cce_fwd(const void* x, const long long* target, const float* weight, float* loss_pos, double* partials,
               float* fwd_out, int N, int K, int S, int ignore_index, float gamma, int dtype, void* stream) {
  if (bad_nks(N, K, S) || (gamma != 0.f && K < 2)) return (int)cudaErrorInvalidValue;  // C divides by K - 1
  CceParams p{};
  p.x = x; p.target = target; p.weight = weight; p.loss_pos = loss_pos; p.partials = partials;
  p.N = N; p.K = K; p.S = S; p.ignore_index = ignore_index; p.gamma = gamma;
  const long long P = (long long)N * S;
  if (P == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = grid_for(P, S == 1 ? kThreads / 32 : kThreads);
#define HB_CCE_FWD(T) cce_kernel<T, false><<<grid, kThreads, 0, st>>>(p)
  HB_LOSS_DTYPE_SWITCH(dtype, HB_CCE_FWD)
#undef HB_CCE_FWD
  HB_LAUNCH_CHECK();
  finalize3_kernel<<<1, 32, 0, st>>>(partials, grid, (double)P, gamma, fwd_out);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_cce_bwd(const void* x, const long long* target, const float* weight, const float* gout, const float* fwd_out,
               void* dx, int N, int K, int S, int ignore_index, float gamma, int reduction, int dtype, void* stream) {
  if (bad_nks(N, K, S) || (gamma != 0.f && K < 2)) return (int)cudaErrorInvalidValue;  // C divides by K - 1
  CceParams p{};
  p.x = x; p.target = target; p.weight = weight; p.gout = gout; p.fwd_out = fwd_out; p.dx = dx;
  p.N = N; p.K = K; p.S = S; p.ignore_index = ignore_index; p.reduction = reduction; p.gamma = gamma;
  const long long P = (long long)N * S;
  if (P == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = grid_for(P, S == 1 ? kThreads / 32 : kThreads);
#define HB_CCE_BWD(T) cce_kernel<T, true><<<grid, kThreads, 0, st>>>(p)
  HB_LOSS_DTYPE_SWITCH(dtype, HB_CCE_BWD)
#undef HB_CCE_BWD
  HB_LAUNCH_CHECK();
  return 0;
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
#define HB_MCL_FWD(T)                                                                                      \
  {                                                                                                        \
    const int vec = S % Vec16<T>::N == 0 && aligned16(x);                                                  \
    mcl_row_lse_kernel<T><<<(unsigned)rows, kThreads, 0, st>>>((const T*)x, S, vec, row_lse);              \
    HB_LAUNCH_CHECK();                                                                                     \
    mcl_fwd_kernel<T><<<grid, kThreads, 0, st>>>(p);                                                       \
  }
  HB_LOSS_DTYPE_SWITCH(dtype, HB_MCL_FWD)
#undef HB_MCL_FWD
  HB_LAUNCH_CHECK();
  finalize3_kernel<<<1, 32, 0, st>>>(partials, grid, (double)P, -alpha, fwd_out);
  HB_LAUNCH_CHECK();
  return 0;
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
#define HB_MCL_BWD(T)                                                                                      \
  {                                                                                                        \
    mcl_rdot_kernel<T><<<(unsigned)groups, rt, smem, st>>>(p);                                             \
    HB_LAUNCH_CHECK();                                                                                     \
    mcl_bwd_kernel<T><<<grid, kThreads, 0, st>>>(p);                                                       \
  }
  HB_LOSS_DTYPE_SWITCH(dtype, HB_MCL_BWD)
#undef HB_MCL_BWD
  HB_LAUNCH_CHECK();
  return 0;
}

#undef HB_LOSS_DTYPE_SWITCH

}  // extern "C"
