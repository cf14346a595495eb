// Squeeze-excite plumbing of the ReXNet blocks (reference holocron/models/classification/rexnet.py:38-66, 112-137):
//   gate-apply + activation:  out[n,p,c] = act(x[n,p,c] * gate[n,c])          (reference: `x * y` then the block's ReLU6)
//   its backward:             dz = dout * act'(x*gate);  dx = dz * gate;  dgate[n,c] = sum_p dz * x
//   global average pooling:   y[n,c] = mean_p x[n,p,c]                          (the squeeze; also the classifier heads)
// NHWC bf16 activations, fp32 gate / accumulation. One CTA per (image, channel slab): the per-image reductions need no
// atomics (deterministic) and 256 images x slabs CTAs fill the GPU. Replaces, per SE block and step, a broadcast multiply,
// an activation pass, two multiplies + a reduction in backward and a one-thread-per-(n, 8 channels) pooling walk.
#include "common.cuh"
#include "act.cuh"
#include "slab.cuh"

namespace {

using namespace hb;

constexpr int kThreads = kSlabThreads;

// grid = (1, slabs, N)
__global__ void __launch_bounds__(kThreads) gate_act_fwd_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gate,
                                                               __nv_bfloat16* __restrict__ out, int HW, int C, int act,
                                                               float slope, SlabGeo g) {
  const auto [tx, ty, cg, active] = g.thread();
  if (!active) return;
  const size_t n = blockIdx.z;
  float gt[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) gt[j] = gate[n * C + cg * 8 + j];
  const __nv_bfloat16* xp = x + n * HW * C + cg * 8;
  __nv_bfloat16* op = out + n * HW * C + cg * 8;
  int r = ty;
  for (; r + g.rows_t < HW; r += 2 * g.rows_t) {   // two rows in flight
    const Vec16<__nv_bfloat16> a = ld16_stream(xp + (size_t)r * C), b = ld16_stream(xp + (size_t)(r + g.rows_t) * C);
    float fa[8], fb[8];
    unpack8(a, fa); unpack8(b, fb);
#pragma unroll
    for (int j = 0; j < 8; ++j) { fa[j] = act_fwd(act, fa[j] * gt[j], slope); fb[j] = act_fwd(act, fb[j] * gt[j], slope); }
    store8(op + (size_t)r * C, fa);
    store8(op + (size_t)(r + g.rows_t) * C, fb);
  }
  if (r < HW) {
    float fa[8];
    unpack8(ld16_stream(xp + (size_t)r * C), fa);
#pragma unroll
    for (int j = 0; j < 8; ++j) fa[j] = act_fwd(act, fa[j] * gt[j], slope);
    store8(op + (size_t)r * C, fa);
  }
}

__global__ void __launch_bounds__(kThreads) gate_act_bwd_kernel(const __nv_bfloat16* __restrict__ dout,
                                                               const __nv_bfloat16* __restrict__ x,
                                                               const float* __restrict__ gate, __nv_bfloat16* __restrict__ dx,
                                                               float* __restrict__ dgate, int HW, int C, int act, float slope,
                                                               SlabGeo g) {
  __shared__ float red[kThreads * 8];
  const auto [tx, ty, cg, active] = g.thread();
  const size_t n = blockIdx.z;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (active) {
    float gt[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) gt[j] = gate[n * C + cg * 8 + j];
    const size_t base = n * HW * C + cg * 8;
    for (int r = ty; r < HW; r += g.rows_t) {
      const Vec16<__nv_bfloat16> xv = ld16_stream(x + base + (size_t)r * C), dv = ld16_stream(dout + base + (size_t)r * C);
      float xf[8], df[8], o[8];
      unpack8(xv, xf); unpack8(dv, df);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float dz = df[j] * act_grad(act, xf[j] * gt[j], slope);
        o[j] = dz * gt[j];
        acc[j] = fmaf(dz, xf[j], acc[j]);
      }
      store8(dx + base + (size_t)r * C, o);
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[threadIdx.x * 8 + j] = acc[j];
  __syncthreads();
  fold_row_lanes<float, 1>(g, red, [&](int c, const float (&a)[1]) { dgate[n * C + c] = a[0]; });
}

// y[n, c] = mean over the HW rows of image n; grid = (1, slabs, N)
__global__ void __launch_bounds__(kThreads) gap_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                          int HW, int C, SlabGeo g) {
  __shared__ float red[kThreads * 8];
  const auto [tx, ty, cg, active] = g.thread();
  const size_t n = blockIdx.z;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (active) {
    const __nv_bfloat16* p = x + n * HW * C + cg * 8;
    int r = ty;
    for (; r + g.rows_t < HW; r += 2 * g.rows_t) {
      const Vec16<__nv_bfloat16> a = ld16_stream(p + (size_t)r * C), b = ld16_stream(p + (size_t)(r + g.rows_t) * C);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += __bfloat162float(a.v[j]) + __bfloat162float(b.v[j]);
    }
    if (r < HW) {
      const Vec16<__nv_bfloat16> a = ld16_stream(p + (size_t)r * C);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += __bfloat162float(a.v[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[threadIdx.x * 8 + j] = acc[j];
  __syncthreads();
  const float inv = 1.f / (float)HW;
  fold_row_lanes<float, 1>(g, red, [&](int c, const float (&a)[1]) { y[n * C + c] = __float2bfloat16_rn(a[0] * inv); });
}

}  // namespace

extern "C" {

int hb_gate_act_fwd_bf16(const void* x, const float* gate, void* out, int N, int HW, int C, int act, float slope,
                         void* stream) {
  if (C % 8 != 0 || act == ACT_FRELU) return (int)cudaErrorInvalidValue;
  if (N <= 0 || HW <= 0) return 0;
  const SlabGeo g = SlabGeo::make(C);
  gate_act_fwd_kernel<<<dim3(1, g.slabs, N), kThreads, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x, gate, (__nv_bfloat16*)out, HW, C, act, slope, g);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_gate_act_bwd_bf16(const void* dout, const void* x, const float* gate, void* dx, float* dgate, int N, int HW, int C,
                         int act, float slope, void* stream) {
  if (C % 8 != 0 || act == ACT_FRELU) return (int)cudaErrorInvalidValue;
  if (N <= 0 || HW <= 0) return 0;
  const SlabGeo g = SlabGeo::make(C);
  gate_act_bwd_kernel<<<dim3(1, g.slabs, N), kThreads, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)dout, (const __nv_bfloat16*)x, gate, (__nv_bfloat16*)dx, dgate, HW, C, act, slope, g);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_gap_fwd_bf16(const void* x, void* y, int N, int HW, int C, void* stream) {
  if (C % 8 != 0) return (int)cudaErrorInvalidValue;
  if (N <= 0 || HW <= 0) return 0;
  const SlabGeo g = SlabGeo::make(C);
  gap_fwd_kernel<<<dim3(1, g.slabs, N), kThreads, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, HW, C, g);
  HB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
