// Device-side control block of a captured training step + gradient clipping, so that the trainer-loop semantics of the
// reference (holocron/trainer/core.py:135-227: NaN-loss skipping :153-159, gradient accumulation and clip_grad_norm_
// :184-208, per-iteration scheduler.step() :161) need no host synchronisation and survive CUDA-graph replay.
//
// ctl (8 x 4 bytes, device): [0] lr (f32)  [1] beta1 (f32, < 0: keep the optimizer's)  [2] skip (i32)  [3] bad (i32)
//                            [4] iter (i32) [5] nan_run (i32)  [6] opt_steps (i32)  [7] grad_norm (f32)
#include "common.cuh"

namespace {

using namespace hb;

struct Ctl { float lr; float beta1; int skip; int bad; int iter; int nan_run; int opt_steps; float grad_norm; };

// after every micro-batch: remember a non-finite loss of the accumulation window
__global__ void ctl_observe_kernel(Ctl* c, const float* loss, int skip_nan) {
  if (skip_nan && !isfinite(*loss)) c->bad = 1;
}

// before the optimizer update: schedule lookup (one entry per ITERATION, like scheduler.step() after every batch) and the
// skip decision of this update; after it (phase 1): counters
__global__ void ctl_step_kernel(Ctl* c, const float* table, int n, int phase) {
  if (phase == 0) {
    if (table && n > 0) {
      const int i = c->iter < n ? c->iter : n - 1;
      c->lr = table[2 * i];
      c->beta1 = table[2 * i + 1];
    }
    c->skip = c->bad;
    c->nan_run = c->bad ? c->nan_run + 1 : 0;
  } else {
    if (!c->skip) c->opt_steps += 1;
    c->bad = 0;
  }
}

__global__ void ctl_tick_kernel(Ctl* c) { c->iter += 1; }

// deterministic two-stage global L2 norm of the flat gradient bucket: per-block partial sums of squares ...
__global__ void __launch_bounds__(256) sumsq_partials_kernel(const float* __restrict__ g, long long n, double* __restrict__ parts) {
  __shared__ double red[32];
  double acc = 0.0;
  const long long n4 = n & ~3LL;
  for (long long i = ((long long)blockIdx.x * 256 + threadIdx.x) * 4; i < n4; i += (long long)gridDim.x * 1024) {
    const float4 v = *reinterpret_cast<const float4*>(g + i);
    acc += (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
  }
  if (blockIdx.x == 0) for (long long i = n4 + threadIdx.x; i < n; i += 256) acc += (double)g[i] * g[i];
  const double tot = block_sum<double>(acc, red);
  if (threadIdx.x == 0) parts[blockIdx.x] = tot;
}

// ... then every block folds the partials in the same fixed order, forms torch's clip coefficient
// min(1, max_norm / (norm + 1e-6)) (torch.nn.utils.clip_grad_norm_) and scales its slice in place. As torch.clamp does,
// the minimum keeps a NaN coefficient: a NaN norm makes every gradient NaN (an inf norm makes them 0, or NaN where inf).
__global__ void __launch_bounds__(256) clip_scale_kernel(float* __restrict__ g, long long n, const double* __restrict__ parts,
                                                         int nparts, float max_norm, Ctl* c) {
  __shared__ float coef_s;
  if (threadIdx.x == 0) {
    double tot = 0.0;
    for (int i = 0; i < nparts; ++i) tot += parts[i];
    const float norm = (float)sqrt(tot);
    float coef = max_norm / (norm + 1e-6f);
    coef_s = coef > 1.f ? 1.f : coef;
    if (blockIdx.x == 0 && c) c->grad_norm = norm;
  }
  __syncthreads();
  const float coef = coef_s;
  if (coef >= 1.f) return;
  const long long n4 = n & ~3LL;
  for (long long i = ((long long)blockIdx.x * 256 + threadIdx.x) * 4; i < n4; i += (long long)gridDim.x * 1024) {
    float4 v = *reinterpret_cast<float4*>(g + i);
    v.x *= coef; v.y *= coef; v.z *= coef; v.w *= coef;
    *reinterpret_cast<float4*>(g + i) = v;
  }
  if (blockIdx.x == 0) for (long long i = n4 + threadIdx.x; i < n; i += 256) g[i] *= coef;
}

}  // namespace

extern "C" {

int hb_train_ctl_bytes(void) { return (int)sizeof(Ctl); }

int hb_train_ctl_observe(void* ctl, const float* loss, int skip_nan, void* stream) {
  ctl_observe_kernel<<<1, 1, 0, (cudaStream_t)stream>>>((Ctl*)ctl, loss, skip_nan);
  HB_LAUNCH_CHECK();
  return 0;
}

// phase 0: before the optimizer update (schedule lookup: table = n x {lr, beta1} fp32 or NULL; skip decision);
// phase 1: after it (counters, window reset)
int hb_train_ctl_step(void* ctl, const float* table, int n, int phase, void* stream) {
  ctl_step_kernel<<<1, 1, 0, (cudaStream_t)stream>>>((Ctl*)ctl, table, n, phase);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_train_ctl_tick(void* ctl, void* stream) {
  ctl_tick_kernel<<<1, 1, 0, (cudaStream_t)stream>>>((Ctl*)ctl);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_grad_clip_partials_max(void) { return HB_NUM_SMS * 4; }

// torch.nn.utils.clip_grad_norm_(params, max_norm) on a flat fp32 gradient buffer: two launches, no host sync, fixed
// summation order. scratch: double [hb_grad_clip_partials_max()]. ctl (optional) receives the norm.
int hb_grad_clip_norm(float* grads, long long n, float max_norm, double* scratch, void* ctl, void* stream) {
  if (!grads || !scratch || n <= 0) return (int)cudaErrorInvalidValue;
  if (!hb::aligned16(grads)) return (int)cudaErrorMisalignedAddress;
  long long want = (n / 4 + 255) / 256;
  int grid = (int)(want < HB_NUM_SMS * 4 ? (want < 1 ? 1 : want) : HB_NUM_SMS * 4);
  sumsq_partials_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(grads, n, scratch);
  HB_LAUNCH_CHECK();
  clip_scale_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(grads, n, scratch, grid, max_norm, (Ctl*)ctl);
  HB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
