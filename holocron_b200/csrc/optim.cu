// Multi-tensor optimizer steps: AdaBelief, LAMB, TAdam, AdamP, Adan, AdEMAMix, LARS, RaLars and the Lookahead weight
// synchronisation (reference holocron/optim/{adabelief,lamb,tadam,adamp,adan,ademamix,lars,ralars,wrapper}.py).
//
// The reference loops over parameter tensors in Python and issues ~9-16 ATen kernels per tensor (plus, for LAMB, LARS,
// RaLars and AdamP, host synchronisations per tensor). Here a device-resident table describes every tensor of a parameter
// group (pointers + numel) and a chunk list maps each CTA to a 4096-element slice of one tensor, so a whole group is
// updated by a fixed number of launches that are 128-bit-vectorised HBM streams (AdaBelief: 28 B/param algorithmic traffic),
// with a scalar path for a tensor any of whose pointers the launch reads or writes is not 16-byte aligned:
//
//   family      launches                                     per-tensor reduction (scratch doubles)   control block
//   AdaBelief   1                                            -                                         read
//   LAMB        2  moments + norms, apply                    ||p||^2, ||update||^2          [2T]      -
//   TAdam       3  reduce, apply, W_t update                 sum (g - m)^2 / (v + eps)      [T]       -
//   AdamP       2  moments + sums, apply                     <p,g>, ||p||^2, ||g||^2, <p,pt> [4T]     read (both passes)
//   Adan        1                                            -                                         read
//   AdEMAMix    1                                            -                                         read
//   LARS        2  norms, apply                              ||p||^2, ||g||^2               [2T]      -
//   RaLars      2  moments + norms, apply                    ||p||^2, ||update||^2          [2T]      -
//   Lookahead   1  (weight synchronisation)                  -                                         -
//
// A reduction has to complete before the update that uses it, hence the extra launches. Parameters, gradients and every
// state tensor are fp32: two moments per tensor, plus the amsgrad maximum (AdaBelief, TAdam, AdamP, Adan), a third moment
// (Adan's exp_avg_delta, AdEMAMix's exp_avg_slow), Adan's prev_grad, the LARS momentum buffer, the Lookahead slow weights,
// and one fp32 scalar per tensor for TAdam's W_t and the LAMB / RaLars trust ratio. Per-tensor reductions are fp32 within a
// thread (at most 16 terms), fp64 from the block reduction on, and added across CTAs with fp64 atomics (order-insensitive
// at fp32 precision). "Control block": the kernel takes the learning rate (and beta1 when >= 0) from the device block of a
// captured training step and does nothing while its skip flag is set (apply_ctl below); the step counter of the families
// that keep one on the device (AdaBelief, AdamP, Adan) does not advance either.
//
// Every kernel is a prologue (control block, table lookup, bias corrections), a list of streams, one element function that
// for_chunk calls on the values of each element, and for the reducing passes chunk_sums.
#include "common.cuh"

namespace {

using namespace hb;

constexpr int kThreads = 256;
constexpr int kChunk = 4096;  // elements per CTA

struct TensorMeta {
  float* p;
  const float* g;
  float* m;
  float* v;
  float* vmax;  // amsgrad state or null
  float* aux;   // TAdam: W_t (1 element); LAMB / RaLars: local_lr out (1 element); Adan: prev_grad (full tensor); else null
  float* ext;   // Adan: exp_avg_delta; AdEMAMix: exp_avg_slow; else null
  long long numel;
};

struct Hyper {
  float lr, beta1, beta2, eps, wd;
  float bc1, bc2;       // bias corrections 1 - beta^step (host-computed) ...
  const int* step_dev;  // ... or, when non-null, computed on device from *step_dev (CUDA-graph friendly)
  int amsgrad;
  float clip_lo, clip_hi;  // LAMB
  float dof;               // TAdam (< 0: use numel)
  float delta;             // AdamP
  float beta3, alpha;      // Adan / AdEMAMix
  float bc3;               // Adan: 1 - beta3^step
  float momentum, dampening;  // LARS
  int nesterov, first;        // LARS: `first` = the momentum buffers of this launch's tensors do not exist yet
  int mode;                   // RaLars: 0 rectified (x r_t), 1 plain Adam ratio, 2 unadapted momentum
  float r_t;                  // RaLars variance rectification
  // optional device control block of a captured training step (train_ctl.cu): {lr, beta1, skip, ...}. When given, the
  // learning rate (and beta1 when >= 0) are read from it and the whole update is skipped while skip != 0
  const float* ctl;
};

// applies the control block to a by-value copy of the hyper-parameters; returns false when the update must be skipped
__device__ __forceinline__ bool apply_ctl(Hyper& h) {
  if (!h.ctl) return true;
  if (reinterpret_cast<const int*>(h.ctl)[2] != 0) return false;
  h.lr = h.ctl[0];
  if (h.ctl[1] >= 0.f) h.beta1 = h.ctl[1];
  return true;
}

__device__ __forceinline__ void bias_corrections(const Hyper& h, float& bc1, float& bc2) {
  if (h.step_dev) {
    const double s = (double)(*h.step_dev);
    bc1 = (float)(1.0 - pow((double)h.beta1, s));
    bc2 = (float)(1.0 - pow((double)h.beta2, s));
  } else {
    bc1 = h.bc1; bc2 = h.bc2;
  }
}

// One tensor the element function sees: each element's value is read from `in` (0 when null) and, after the function
// has run, written to `out` (not at all when null). `v` holds the values in flight, one per lane on the vector path.
struct Stream {
  const float* in;
  float* out;
  float4 v;

  __device__ __forceinline__ bool vec_ok() const { return aligned16(in) && aligned16(out); }
  __device__ __forceinline__ void load4(long long i) {
    v = in ? *reinterpret_cast<const float4*>(in + i) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  __device__ __forceinline__ void store4(long long i) const { if (out) *reinterpret_cast<float4*>(out + i) = v; }
  __device__ __forceinline__ void load1(long long i) { v.x = in ? in[i] : 0.f; }
  __device__ __forceinline__ void store1(long long i) const { if (out) out[i] = v.x; }
};

__device__ __forceinline__ Stream rd(const float* t) { return {t, nullptr}; }
__device__ __forceinline__ Stream rw(float* t) { return {t, t}; }

// Chunk walker: calls f with one float& per stream, in the order the streams are given, for each element of this CTA's
// chunk. Four elements at a time (lanes x, y, z, w in that order) when every non-null pointer of the streams is 16-byte
// aligned, one at a time otherwise and for the tail.
template <typename F, typename... S>
__device__ __forceinline__ void for_chunk(long long numel, int chunk, F f, S... s) {
  const long long base = (long long)chunk * kChunk;
  const long long end = min(base + (long long)kChunk, numel);
  long long i = base + threadIdx.x;
  if ((s.vec_ok() && ...)) {
    const long long end4 = base + ((end - base) & ~3LL);
    for (long long j = base + threadIdx.x * 4; j < end4; j += kThreads * 4) {
      (s.load4(j), ...);
      f(s.v.x...);
      f(s.v.y...);
      f(s.v.z...);
      f(s.v.w...);
      (s.store4(j), ...);
    }
    i = end4 + threadIdx.x;
  }
  for (; i < end; i += kThreads) {
    (s.load1(i), ...);
    f(s.v.x...);
    (s.store1(i), ...);
  }
}

// Per-tensor sums of this CTA: K block reductions in fp64, then thread 0 adds them into row[0..K) with fp64 atomics.
template <int K>
__device__ __forceinline__ void chunk_sums(const float (&acc)[K], double* row) {
  __shared__ double red[32];
  double tot[K];
#pragma unroll
  for (int k = 0; k < K; ++k) tot[k] = block_sum<double>((double)acc[k], red);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) atomicAdd(&row[k], tot[k]);
  }
}

// ---------------------------------------------------------------------------------------------------
// AdaBelief  (reference adabelief.py:121-167; NB no +eps inside the belief EMA)
__global__ void __launch_bounds__(kThreads) adabelief_kernel(const TensorMeta* __restrict__ metas,
                                                             const int2* __restrict__ chunks, Hyper h) {
  if (!apply_ctl(h)) return;
  const int2 c = chunks[blockIdx.x];
  const TensorMeta t = metas[c.x];
  float bc1, bc2;
  bias_corrections(h, bc1, bc2);
  const float step_size = h.lr / bc1;
  const float inv_sqrt_bc2 = 1.f / sqrtf(bc2);
  const bool ams = h.amsgrad && t.vmax;
  auto one = [&](float& p, float g, float& m, float& s, float& x) {
    if (h.wd != 0.f) g = fmaf(h.wd, p, g);
    m = fmaf(1.f - h.beta1, g, h.beta1 * m);
    const float r = g - m;
    s = fmaf(1.f - h.beta2, r * r, h.beta2 * s);
    float sec = s;
    if (ams) { x = fmaxf(x, s); sec = x; }
    const float denom = sqrtf(sec) * inv_sqrt_bc2 + h.eps;
    p = p - step_size * (m / denom);
  };
  for_chunk(t.numel, c.y, one, rw(t.p), rd(t.g), rw(t.m), rw(t.v), rw(ams ? t.vmax : nullptr));
}

// ---------------------------------------------------------------------------------------------------
// LAMB (reference lamb.py:79-137): no bias correction; update = m/(sqrt(v)+eps) + wd*p;
// local_lr = clamp(||p||, lo, hi) / ||update||  (1 when either norm is 0)
__global__ void __launch_bounds__(kThreads) lamb_moments_kernel(const TensorMeta* __restrict__ metas,
                                                                const int2* __restrict__ chunks, Hyper h,
                                                                double* __restrict__ norms /*[T][2]*/) {
  const int2 c = chunks[blockIdx.x];
  const TensorMeta t = metas[c.x];
  float pn = 0.f, un = 0.f;   // <= 16 elements per thread: fp32 partials, fp64 from the block reduction on
  auto one = [&](float p, float g, float& m, float& v) {
    m = fmaf(1.f - h.beta1, g, h.beta1 * m);
    v = fmaf(1.f - h.beta2, g * g, h.beta2 * v);
    float u = m / (sqrtf(v) + h.eps);
    if (h.wd != 0.f) u = fmaf(h.wd, p, u);
    pn = fmaf(p, p, pn);
    un = fmaf(u, u, un);
  };
  for_chunk(t.numel, c.y, one, rd(t.p), rd(t.g), rw(t.m), rw(t.v));
  chunk_sums<2>({pn, un}, norms + 2 * c.x);
}

__global__ void __launch_bounds__(kThreads) lamb_apply_kernel(const TensorMeta* __restrict__ metas,
                                                              const int2* __restrict__ chunks, Hyper h,
                                                              const double* __restrict__ norms) {
  const int2 c = chunks[blockIdx.x];
  const TensorMeta t = metas[c.x];
  const float p_norm = (float)sqrt(norms[2 * c.x + 0]);
  const float u_norm = (float)sqrt(norms[2 * c.x + 1]);
  const float phi = fminf(fmaxf(p_norm, h.clip_lo), h.clip_hi);
  const float local_lr = (phi == 0.f || u_norm == 0.f) ? 1.f : phi / u_norm;
  if (c.y == 0 && threadIdx.x == 0 && t.aux) *t.aux = local_lr;
  const float a = h.lr * local_lr;
  auto one = [&](float& p, float m, float v) {
    float u = m / (sqrtf(v) + h.eps);
    if (h.wd != 0.f) u = fmaf(h.wd, p, u);
    p = p - a * u;
  };
  for_chunk(t.numel, c.y, one, rw(t.p), rd(t.m), rd(t.v));
}

// ---------------------------------------------------------------------------------------------------
// AdamP (reference adamp.py:144-191): Adam moments with bias correction; when the gradient is (nearly) orthogonal to
// the weight tensor, cos(p, g) < delta / sqrt(numel), the radial component of the update is projected out:
//   pt = (m / bc1) / (sqrt(v) / sqrt(bc2) + eps);  pt -= <p / (||p|| + eps), pt> * p / (||p|| + eps);  p -= lr * pt
// Pass 1 updates the moments and reduces <p,g>, ||p||^2, ||g||^2, <p,pt> per tensor; pass 2 applies (40 B / parameter).
__device__ __forceinline__ float adamp_pt(float m, float v, float vmax_or_neg, float bc1, float inv_sqrt_bc2, float eps) {
  const float sec = vmax_or_neg >= 0.f ? vmax_or_neg : v;
  return (m / bc1) / (sqrtf(sec) * inv_sqrt_bc2 + eps);
}

__global__ void __launch_bounds__(kThreads) adamp_moments_kernel(const TensorMeta* __restrict__ metas,
                                                                 const int2* __restrict__ chunks, Hyper h,
                                                                 double* __restrict__ sums /*[T][4]*/) {
  if (!apply_ctl(h)) return;
  const int2 c = chunks[blockIdx.x];
  const TensorMeta t = metas[c.x];
  float bc1, bc2;
  bias_corrections(h, bc1, bc2);
  const float inv_sqrt_bc2 = 1.f / sqrtf(bc2);
  const bool ams = h.amsgrad && t.vmax;
  float s_pg = 0.f, s_pp = 0.f, s_gg = 0.f, s_ppt = 0.f;
  auto one = [&](float p, float g, float& m, float& v, float& x) {
    if (h.wd != 0.f) g = fmaf(h.wd, p, g);
    m = fmaf(1.f - h.beta1, g, h.beta1 * m);
    v = fmaf(1.f - h.beta2, g * g, h.beta2 * v);
    if (ams) x = fmaxf(x, v);
    const float pt = adamp_pt(m, v, ams ? x : -1.f, bc1, inv_sqrt_bc2, h.eps);
    s_pg = fmaf(p, g, s_pg); s_pp = fmaf(p, p, s_pp); s_gg = fmaf(g, g, s_gg); s_ppt = fmaf(p, pt, s_ppt);
  };
  for_chunk(t.numel, c.y, one, rd(t.p), rd(t.g), rw(t.m), rw(t.v), rw(ams ? t.vmax : nullptr));
  chunk_sums<4>({s_pg, s_pp, s_gg, s_ppt}, sums + 4 * c.x);
}

__global__ void __launch_bounds__(kThreads) adamp_apply_kernel(const TensorMeta* __restrict__ metas,
                                                               const int2* __restrict__ chunks, Hyper h,
                                                               const double* __restrict__ sums) {
  if (!apply_ctl(h)) return;
  const int2 c = chunks[blockIdx.x];
  const TensorMeta t = metas[c.x];
  float bc1, bc2;
  bias_corrections(h, bc1, bc2);
  const float inv_sqrt_bc2 = 1.f / sqrtf(bc2);
  const bool ams = h.amsgrad && t.vmax;
  // F.cosine_similarity clamps each norm at 1e-8 (torch eps default)
  const float pn = (float)sqrt(sums[4 * c.x + 1]), gn = (float)sqrt(sums[4 * c.x + 2]);
  const float cosv = (float)sums[4 * c.x + 0] / (fmaxf(pn, 1e-8f) * fmaxf(gn, 1e-8f));
  const bool project = cosv < h.delta / sqrtf((float)t.numel);
  const float inv = 1.f / (pn + h.eps);
  const float k = project ? (float)sums[4 * c.x + 3] * inv * inv : 0.f;   // <p_hat, pt> / (||p|| + eps)
  auto one = [&](float& p, float m, float v, float x) {
    float pt = adamp_pt(m, v, ams ? x : -1.f, bc1, inv_sqrt_bc2, h.eps);
    pt = fmaf(-k, p, pt);
    p = fmaf(-h.lr, pt, p);
  };
  for_chunk(t.numel, c.y, one, rw(t.p), rd(t.m), rd(t.v), rd(ams ? t.vmax : nullptr));
}

// ---------------------------------------------------------------------------------------------------
// TAdam (reference tadam.py:160-212)
__global__ void __launch_bounds__(kThreads) tadam_reduce_kernel(const TensorMeta* __restrict__ metas,
                                                                const int2* __restrict__ chunks, Hyper h,
                                                                double* __restrict__ sums /*[T]*/) {
  const int2 c = chunks[blockIdx.x];
  const TensorMeta t = metas[c.x];
  float acc = 0.f;
  auto one = [&](float p, float g, float m, float v) {
    if (h.wd != 0.f) g = fmaf(h.wd, p, g);
    const float d = g - m;
    acc += (d * d) / (v + h.eps);
  };
  for_chunk(t.numel, c.y, one, rd(h.wd != 0.f ? t.p : nullptr), rd(t.g), rd(t.m), rd(t.v));
  chunk_sums<1>({acc}, sums + c.x);
}

__device__ __forceinline__ float tadam_wt(const TensorMeta& t, const Hyper& h, double sum) {
  const float n = (float)t.numel;
  const float dof = h.dof < 0.f ? n : h.dof;
  return (dof + n) / ((float)sum + dof);
}

__global__ void __launch_bounds__(kThreads) tadam_apply_kernel(const TensorMeta* __restrict__ metas,
                                                               const int2* __restrict__ chunks, Hyper h,
                                                               const double* __restrict__ sums) {
  const int2 c = chunks[blockIdx.x];
  const TensorMeta t = metas[c.x];
  float bc1, bc2;
  bias_corrections(h, bc1, bc2);
  const float step_size = h.lr / bc1;
  const float inv_sqrt_bc2 = 1.f / sqrtf(bc2);
  const float w = tadam_wt(t, h, sums[c.x]);
  const float W = *t.aux;
  const float a = W / (W + w);
  const bool ams = h.amsgrad && t.vmax;
  auto one = [&](float& p, float g, float& m, float& v, float& x) {
    if (h.wd != 0.f) g = fmaf(h.wd, p, g);
    m = m * a + (w * g) / (W + w);
    v = fmaf(1.f - h.beta2, g * g, h.beta2 * v);
    float sec = v;
    if (ams) { x = fmaxf(x, v); sec = x; }
    const float denom = sqrtf(sec) * inv_sqrt_bc2 + h.eps;
    p = p - step_size * (m / denom);
  };
  for_chunk(t.numel, c.y, one, rw(t.p), rd(t.g), rw(t.m), rw(t.v), rw(ams ? t.vmax : nullptr));
}

// W_t <- W_t * (2 beta1 - 1) / beta1 + w_t   (after every CTA of the apply pass has read the old W_t)
__global__ void tadam_wt_update_kernel(const TensorMeta* __restrict__ metas, int T, Hyper h,
                                       const double* __restrict__ sums) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T) return;
  const TensorMeta t = metas[i];
  const float w = tadam_wt(t, h, sums[i]);
  *t.aux = *t.aux * ((2.f * h.beta1 - 1.f) / h.beta1) + w;
}

// ---------------------------------------------------------------------------------------------------
// Adan (reference adan.py:145-199). Quirks kept: `prev_grad` is read but never written by the reference (it stays at its
// initial zeros, so delta_grad == grad unless a loaded state says otherwise); the update mixes beta2 * exp_avg_sq / bc2
// (not 1 - beta2); with weight decay the parameter is divided by (1 + wd * lr) after the step.
// m = exp_avg, v = exp_avg_sq (EMA of gradient differences), ext = exp_avg_delta (EMA of squares), vmax = its running max.
__global__ void __launch_bounds__(kThreads) adan_kernel(const TensorMeta* __restrict__ metas, const int2* __restrict__ chunks,
                                                        Hyper h) {
  if (!apply_ctl(h)) return;
  const int2 c = chunks[blockIdx.x];
  const TensorMeta t = metas[c.x];
  float bc1, bc2, bc3 = h.bc3;
  bias_corrections(h, bc1, bc2);
  if (h.step_dev) bc3 = (float)(1.0 - pow((double)h.beta3, (double)(*h.step_dev)));
  const float inv_sqrt_bc3 = 1.f / sqrtf(bc3);
  const bool ams = h.amsgrad && t.vmax;
  const float shrink = 1.f + h.wd * h.lr;
  auto one = [&](float& p, float g, float pg, float& m, float& v, float& n, float& x) {
    if (h.wd != 0.f) g = fmaf(h.wd, p, g);
    m = fmaf(1.f - h.beta1, g, h.beta1 * m);
    const float dg = g - pg;
    v = fmaf(1.f - h.beta2, dg, h.beta2 * v);
    const float tmp = fmaf(h.beta2, dg, g);
    n = fmaf(1.f - h.beta3, tmp * tmp, h.beta3 * n);
    float sec = n;
    if (ams) { x = fmaxf(x, n); sec = x; }
    const float denom = sqrtf(sec) * inv_sqrt_bc3 + h.eps;
    const float pt = (m / bc1 + h.beta2 * v / bc2) / denom;
    p = fmaf(-h.lr, pt, p);
    if (h.wd != 0.f) p = p / shrink;
  };
  for_chunk(t.numel, c.y, one, rw(t.p), rd(t.g), rd(t.aux), rw(t.m), rw(t.v), rw(t.ext), rw(ams ? t.vmax : nullptr));
}

// ---------------------------------------------------------------------------------------------------
// AdEMAMix (reference ademamix.py:138-176): fast EMA m1 (bias-corrected), slow EMA m2 (beta3, not corrected), Adam second
// moment; p -= lr * (m1 / bc1 + alpha * m2) / (sqrt(nu) / sqrt(bc2) + eps). m = exp_avg, ext = exp_avg_slow, v = exp_avg_sq.
__global__ void __launch_bounds__(kThreads) ademamix_kernel(const TensorMeta* __restrict__ metas,
                                                            const int2* __restrict__ chunks, Hyper h) {
  if (!apply_ctl(h)) return;
  const int2 c = chunks[blockIdx.x];
  const TensorMeta t = metas[c.x];
  float bc1, bc2;
  bias_corrections(h, bc1, bc2);
  const float inv_sqrt_bc2 = 1.f / sqrtf(bc2);
  auto one = [&](float& p, float g, float& m1, float& m2, float& nu) {
    if (h.wd != 0.f) g = fmaf(h.wd, p, g);
    m1 = fmaf(1.f - h.beta1, g, h.beta1 * m1);
    nu = fmaf(1.f - h.beta2, g * g, h.beta2 * nu);
    m2 = fmaf(1.f - h.beta3, g, h.beta3 * m2);
    const float denom = sqrtf(nu) * inv_sqrt_bc2 + h.eps;
    p = fmaf(-h.lr, fmaf(h.alpha, m2, m1 / bc1) / denom, p);
  };
  for_chunk(t.numel, c.y, one, rw(t.p), rd(t.g), rw(t.m), rw(t.ext), rw(t.v));
}

// ---------------------------------------------------------------------------------------------------
// LARS (reference lars.py:91-135): local_lr = ||p|| / (||g|| + wd ||p||) (1 when either is 0; `scale_clip` is stored but never
// applied by the reference); d_p = g + wd * p is written back INTO THE GRADIENT like the reference's in-place add_;
// SGD momentum with dampening / Nesterov, the first buffer being a copy of d_p. m = momentum_buffer (may be null).
__global__ void __launch_bounds__(kThreads) lars_norms_kernel(const TensorMeta* __restrict__ metas,
                                                              const int2* __restrict__ chunks, double* __restrict__ norms) {
  const int2 c = chunks[blockIdx.x];
  const TensorMeta t = metas[c.x];
  float pn = 0.f, gn = 0.f;
  auto one = [&](float p, float g) {
    pn = fmaf(p, p, pn);
    gn = fmaf(g, g, gn);
  };
  for_chunk(t.numel, c.y, one, rd(t.p), rd(t.g));
  chunk_sums<2>({pn, gn}, norms + 2 * c.x);
}

__global__ void __launch_bounds__(kThreads) lars_apply_kernel(const TensorMeta* __restrict__ metas,
                                                              const int2* __restrict__ chunks, Hyper h,
                                                              const double* __restrict__ norms) {
  const int2 c = chunks[blockIdx.x];
  const TensorMeta t = metas[c.x];
  const float p_norm = (float)sqrt(norms[2 * c.x + 0]);
  float denom = (float)sqrt(norms[2 * c.x + 1]);
  if (h.wd != 0.f) denom = fmaf(h.wd, p_norm, denom);
  const float local_lr = (p_norm == 0.f || denom == 0.f) ? 1.f : p_norm / denom;
  const float a = h.lr * local_lr;
  const bool mom = h.momentum != 0.f && t.m != nullptr;
  auto one = [&](float& p, float& g, float& b) {
    if (h.wd != 0.f) g = fmaf(h.wd, p, g);
    float d = g;
    if (mom) {
      b = h.first ? g : fmaf(h.momentum, b, (1.f - h.dampening) * g);
      d = h.nesterov ? fmaf(h.momentum, b, g) : b;
    }
    p = fmaf(-a, d, p);
  };
  const Stream grad{t.g, h.wd != 0.f ? const_cast<float*>(t.g) : nullptr};
  const Stream buf{mom && !h.first ? t.m : nullptr, mom ? t.m : nullptr};
  for_chunk(t.numel, c.y, one, rw(t.p), grad, buf);
}

// ---------------------------------------------------------------------------------------------------
// RaLars (reference ralars.py:56-140): RAdam update (rectified / plain Adam ratio / unadapted momentum, chosen on the host
// from the SMA length) + wd * p, scaled by the LARS trust ratio clamp(||p||, *scale_clip) / ||update||.
__device__ __forceinline__ float ralars_update(float p, float m, float v, const Hyper& h, float bc1, float bc2) {
  float u;
  if (h.mode == 2) u = m / bc1;
  else u = h.r_t * ((m / bc1) / (sqrtf(v / bc2) + h.eps));
  if (h.wd != 0.f) u = fmaf(h.wd, p, u);
  return u;
}

// 6 CTAs per SM (<= 40 registers): left to itself ptxas takes 46 (nvcc 12.9), which leaves room for 5
__global__ void __launch_bounds__(kThreads, 6) ralars_moments_kernel(const TensorMeta* __restrict__ metas,
                                                                     const int2* __restrict__ chunks, Hyper h,
                                                                     double* __restrict__ norms) {
  const int2 c = chunks[blockIdx.x];
  const TensorMeta t = metas[c.x];
  float pn = 0.f, un = 0.f;
  auto one = [&](float p, float g, float& m, float& v) {
    m = fmaf(1.f - h.beta1, g, h.beta1 * m);
    v = fmaf(1.f - h.beta2, g * g, h.beta2 * v);
    const float u = ralars_update(p, m, v, h, h.bc1, h.bc2);
    pn = fmaf(p, p, pn);
    un = fmaf(u, u, un);
  };
  for_chunk(t.numel, c.y, one, rd(t.p), rd(t.g), rw(t.m), rw(t.v));
  chunk_sums<2>({pn, un}, norms + 2 * c.x);
}

__global__ void __launch_bounds__(kThreads) ralars_apply_kernel(const TensorMeta* __restrict__ metas,
                                                                const int2* __restrict__ chunks, Hyper h,
                                                                const double* __restrict__ norms) {
  const int2 c = chunks[blockIdx.x];
  const TensorMeta t = metas[c.x];
  const float p_norm = (float)sqrt(norms[2 * c.x + 0]);
  const float u_norm = (float)sqrt(norms[2 * c.x + 1]);
  const float phi = fminf(fmaxf(p_norm, h.clip_lo), h.clip_hi);
  const float local_lr = (phi == 0.f || u_norm == 0.f) ? 1.f : phi / u_norm;
  if (c.y == 0 && threadIdx.x == 0 && t.aux) *t.aux = local_lr;
  const float a = h.lr * local_lr;
  auto one = [&](float& p, float m, float v) { p = fmaf(-a, ralars_update(p, m, v, h, h.bc1, h.bc2), p); };
  for_chunk(t.numel, c.y, one, rw(t.p), rd(t.m), rd(t.v));
}

// ---------------------------------------------------------------------------------------------------
// Lookahead.sync_params (reference wrapper.py:122-135): slow += rate * (fast - slow) (skipped when rate == 0); fast = slow.
// p = fast weights, m = slow weights.
__global__ void __launch_bounds__(kThreads) lookahead_sync_kernel(const TensorMeta* __restrict__ metas,
                                                                  const int2* __restrict__ chunks, float rate) {
  const int2 c = chunks[blockIdx.x];
  const TensorMeta t = metas[c.x];
  auto one = [&](float& f, float& s) {
    s = rate > 0.f ? fmaf(rate, f - s, s) : s;
    f = s;
  };
  for_chunk(t.numel, c.y, one, rw(t.p), rw(t.m));
}

__global__ void step_increment_kernel(int* step, const int* ctl) { if (!ctl || ctl[2] == 0) *step += 1; }

Hyper make_hyper(float lr, float b1, float b2, float eps, float wd, int step, const int* step_dev, int amsgrad) {
  Hyper h{};
  h.lr = lr; h.beta1 = b1; h.beta2 = b2; h.eps = eps; h.wd = wd;
  h.bc1 = (float)(1.0 - pow((double)b1, (double)step));
  h.bc2 = (float)(1.0 - pow((double)b2, (double)step));
  h.step_dev = step_dev;
  h.amsgrad = amsgrad;
  h.dof = -1.f;
  h.delta = 0.1f;
  h.beta3 = 0.f; h.alpha = 0.f; h.bc3 = 1.f;
  h.momentum = 0.f; h.dampening = 0.f; h.nesterov = 0; h.first = 0;
  h.mode = 0; h.r_t = 1.f;
  h.ctl = nullptr;
  return h;
}

}  // namespace

extern "C" {

// metas: device array of T records {p, g, m, v, vmax, aux, ext, numel} (8 x 8 bytes); chunks: device int2[num_chunks]
// {tensor index, chunk index} with chunk = 4096 elements.
int hb_optim_chunk_elems(void) { return kChunk; }

int hb_adabelief_step(const void* metas, const void* chunks, int num_chunks, float lr, float beta1, float beta2,
                      float eps, float weight_decay, int amsgrad, int step, const int* step_dev, const void* ctl,
                      void* stream) {
  if (num_chunks <= 0) return 0;
  Hyper h = make_hyper(lr, beta1, beta2, eps, weight_decay, step, step_dev, amsgrad);
  h.ctl = (const float*)ctl;
  adabelief_kernel<<<num_chunks, kThreads, 0, (cudaStream_t)stream>>>((const TensorMeta*)metas, (const int2*)chunks, h);
  HB_LAUNCH_CHECK();
  return 0;
}

// scratch: device double[2*T], zeroed here. local_lr lands in each tensor's aux slot (if non-null).
int hb_lamb_step(const void* metas, const void* chunks, int num_chunks, int T, float lr, float beta1, float beta2,
                 float eps, float weight_decay, float clip_lo, float clip_hi, double* scratch, void* stream) {
  if (num_chunks <= 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  Hyper h = make_hyper(lr, beta1, beta2, eps, weight_decay, 1, nullptr, 0);
  h.clip_lo = clip_lo; h.clip_hi = clip_hi;
  cudaError_t e = cudaMemsetAsync(scratch, 0, sizeof(double) * 2 * T, st);
  if (e != cudaSuccess) return (int)e;
  lamb_moments_kernel<<<num_chunks, kThreads, 0, st>>>((const TensorMeta*)metas, (const int2*)chunks, h, scratch);
  HB_LAUNCH_CHECK();
  lamb_apply_kernel<<<num_chunks, kThreads, 0, st>>>((const TensorMeta*)metas, (const int2*)chunks, h, scratch);
  HB_LAUNCH_CHECK();
  return 0;
}

// scratch: device double[T], zeroed here. aux = W_t (1-element fp32 state) per tensor. dof < 0 -> numel.
int hb_tadam_step(const void* metas, const void* chunks, int num_chunks, int T, float lr, float beta1, float beta2,
                  float eps, float weight_decay, int amsgrad, float dof, int step, const int* step_dev, double* scratch,
                  void* stream) {
  if (num_chunks <= 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  Hyper h = make_hyper(lr, beta1, beta2, eps, weight_decay, step, step_dev, amsgrad);
  h.dof = dof;
  cudaError_t e = cudaMemsetAsync(scratch, 0, sizeof(double) * T, st);
  if (e != cudaSuccess) return (int)e;
  tadam_reduce_kernel<<<num_chunks, kThreads, 0, st>>>((const TensorMeta*)metas, (const int2*)chunks, h, scratch);
  HB_LAUNCH_CHECK();
  tadam_apply_kernel<<<num_chunks, kThreads, 0, st>>>((const TensorMeta*)metas, (const int2*)chunks, h, scratch);
  HB_LAUNCH_CHECK();
  tadam_wt_update_kernel<<<(T + 127) / 128, 128, 0, st>>>((const TensorMeta*)metas, T, h, scratch);
  HB_LAUNCH_CHECK();
  return 0;
}

// scratch: device double[4*T], zeroed here. delta: projection threshold (reference default 0.1).
int hb_adamp_step(const void* metas, const void* chunks, int num_chunks, int T, float lr, float beta1, float beta2, float eps,
                  float weight_decay, int amsgrad, float delta, int step, const int* step_dev, const void* ctl,
                  double* scratch, void* stream) {
  if (num_chunks <= 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  Hyper h = make_hyper(lr, beta1, beta2, eps, weight_decay, step, step_dev, amsgrad);
  h.delta = delta;
  h.ctl = (const float*)ctl;
  cudaError_t e = cudaMemsetAsync(scratch, 0, sizeof(double) * 4 * T, st);
  if (e != cudaSuccess) return (int)e;
  adamp_moments_kernel<<<num_chunks, kThreads, 0, st>>>((const TensorMeta*)metas, (const int2*)chunks, h, scratch);
  HB_LAUNCH_CHECK();
  adamp_apply_kernel<<<num_chunks, kThreads, 0, st>>>((const TensorMeta*)metas, (const int2*)chunks, h, scratch);
  HB_LAUNCH_CHECK();
  return 0;
}

// Adan: aux = prev_grad, ext = exp_avg_delta, vmax = max_exp_avg_delta (amsgrad). One launch, 40 B / parameter.
int hb_adan_step(const void* metas, const void* chunks, int num_chunks, float lr, float beta1, float beta2, float beta3,
                 float eps, float weight_decay, int amsgrad, int step, const int* step_dev, const void* ctl, void* stream) {
  if (num_chunks <= 0) return 0;
  Hyper h = make_hyper(lr, beta1, beta2, eps, weight_decay, step, step_dev, amsgrad);
  h.beta3 = beta3;
  h.bc3 = (float)(1.0 - pow((double)beta3, (double)step));
  h.ctl = (const float*)ctl;
  adan_kernel<<<num_chunks, kThreads, 0, (cudaStream_t)stream>>>((const TensorMeta*)metas, (const int2*)chunks, h);
  HB_LAUNCH_CHECK();
  return 0;
}

// AdEMAMix: ext = exp_avg_slow. One launch, 36 B / parameter.
int hb_ademamix_step(const void* metas, const void* chunks, int num_chunks, float lr, float beta1, float beta2, float beta3,
                     float alpha, float eps, float weight_decay, int step, const int* step_dev, const void* ctl,
                     void* stream) {
  if (num_chunks <= 0) return 0;
  Hyper h = make_hyper(lr, beta1, beta2, eps, weight_decay, step, step_dev, 0);
  h.beta3 = beta3; h.alpha = alpha;
  h.ctl = (const float*)ctl;
  ademamix_kernel<<<num_chunks, kThreads, 0, (cudaStream_t)stream>>>((const TensorMeta*)metas, (const int2*)chunks, h);
  HB_LAUNCH_CHECK();
  return 0;
}

// LARS: m = momentum buffer (null when momentum == 0); first != 0: the buffers are being created by this step.
// scratch: device double[2*T], zeroed here. With weight decay the gradient tensors are overwritten by g + wd * p.
int hb_lars_step(const void* metas, const void* chunks, int num_chunks, int T, float lr, float momentum, float dampening,
                 float weight_decay, int nesterov, int first, double* scratch, void* stream) {
  if (num_chunks <= 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  Hyper h = make_hyper(lr, 0.f, 0.f, 0.f, weight_decay, 1, nullptr, 0);
  h.momentum = momentum; h.dampening = dampening; h.nesterov = nesterov; h.first = first;
  cudaError_t e = cudaMemsetAsync(scratch, 0, sizeof(double) * 2 * T, st);
  if (e != cudaSuccess) return (int)e;
  lars_norms_kernel<<<num_chunks, kThreads, 0, st>>>((const TensorMeta*)metas, (const int2*)chunks, scratch);
  HB_LAUNCH_CHECK();
  lars_apply_kernel<<<num_chunks, kThreads, 0, st>>>((const TensorMeta*)metas, (const int2*)chunks, h, scratch);
  HB_LAUNCH_CHECK();
  return 0;
}

// RaLars: mode 0 rectified (update x r_t), 1 plain Adam ratio, 2 unadapted momentum; aux = local_lr out (1 element).
// scratch: device double[2*T], zeroed here.
int hb_ralars_step(const void* metas, const void* chunks, int num_chunks, int T, float lr, float beta1, float beta2, float eps,
                   float weight_decay, float clip_lo, float clip_hi, int mode, float r_t, int step, double* scratch,
                   void* stream) {
  if (num_chunks <= 0) return 0;
  if (mode < 0 || mode > 2) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  Hyper h = make_hyper(lr, beta1, beta2, eps, weight_decay, step, nullptr, 0);
  h.clip_lo = clip_lo; h.clip_hi = clip_hi;
  h.mode = mode; h.r_t = mode == 0 ? r_t : 1.f;
  cudaError_t e = cudaMemsetAsync(scratch, 0, sizeof(double) * 2 * T, st);
  if (e != cudaSuccess) return (int)e;
  ralars_moments_kernel<<<num_chunks, kThreads, 0, st>>>((const TensorMeta*)metas, (const int2*)chunks, h, scratch);
  HB_LAUNCH_CHECK();
  ralars_apply_kernel<<<num_chunks, kThreads, 0, st>>>((const TensorMeta*)metas, (const int2*)chunks, h, scratch);
  HB_LAUNCH_CHECK();
  return 0;
}

// Lookahead.sync_params: p = fast weights, m = slow weights
int hb_lookahead_sync(const void* metas, const void* chunks, int num_chunks, float sync_rate, void* stream) {
  if (num_chunks <= 0) return 0;
  lookahead_sync_kernel<<<num_chunks, kThreads, 0, (cudaStream_t)stream>>>((const TensorMeta*)metas, (const int2*)chunks,
                                                                          sync_rate);
  HB_LAUNCH_CHECK();
  return 0;
}

// ctl (optional): control block of a captured training step - the counter only advances when the update is not skipped
int hb_step_increment(int* step_dev, const void* ctl, void* stream) {
  step_increment_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(step_dev, (const int*)ctl);
  HB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
