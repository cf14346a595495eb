// Activation codes shared by the fused BatchNorm / gate kernels: forward value and derivative w.r.t. the pre-activation.
#pragma once
#include <cuda_runtime.h>
#include "common.cuh"

namespace hb {

// ACT_FRELU: out = max(z, residual) with z the normalised branch sum (funnel activation, reference activation.py:58-82)
enum Act { ACT_NONE = 0, ACT_RELU = 1, ACT_RELU6 = 2, ACT_SILU = 3, ACT_LEAKY = 4, ACT_MISH = 5, ACT_HARDMISH = 6, ACT_FRELU = 7 };

// Fast-math forms (the BatchNorm / gate passes are HBM streams: with IEEE division, log1pf and tanhf the SiLU / Mish
// variants are ALU-bound instead). Relative error ~1e-6, far below bf16.
//   sigmoid(z) = 1 / (1 + e^-z)
//   mish(z)    = z * tanh(log(1 + e^z)) = z * n / (n + 2),  n = e^z (e^z + 2)        (tanh(log u) = (u^2-1)/(u^2+1))
__device__ __forceinline__ float fast_sigmoid(float z) { return __fdividef(1.f, 1.f + __expf(-z)); }
__device__ __forceinline__ float mish_tanh_sp(float z) {   // tanh(softplus(z)); -> 1 for large z (e^z overflows past 88)
  if (z > 20.f) return 1.f;
  const float e = __expf(z);
  const float n = e * (e + 2.f);
  return __fdividef(n, n + 2.f);
}

__device__ __forceinline__ float act_fwd(int act, float z, float slope) {
  switch (act) {
    case ACT_RELU: return relu_nan(z);
    case ACT_RELU6: return clamp_nan(z, 0.f, 6.f);
    case ACT_SILU: return z * fast_sigmoid(z);
    case ACT_LEAKY: return z > 0.f ? z : z * slope;
    case ACT_MISH: return z * mish_tanh_sp(z);
    case ACT_HARDMISH: return (0.5f * z) * clamp_nan(z + 2.f, 0.f, 2.f);
    default: return z;
  }
}
__device__ __forceinline__ float act_grad(int act, float z, float slope) {
  switch (act) {
    case ACT_RELU: return z > 0.f ? 1.f : 0.f;
    case ACT_RELU6: return (z > 0.f && z < 6.f) ? 1.f : 0.f;
    case ACT_SILU: {
      const float s = fast_sigmoid(z);
      return s * (1.f + z * (1.f - s));
    }
    case ACT_LEAKY: return z > 0.f ? 1.f : slope;
    case ACT_MISH: {
      const float t = mish_tanh_sp(z);
      const float sg = fast_sigmoid(z);
      return t + z * (1.f - t * t) * sg;
    }
    case ACT_HARDMISH: {
      float t = z + 2.f;
      float c = fminf(fmaxf(t, 0.f), 2.f);
      return 0.5f * c + ((t >= 0.f && t <= 2.f) ? 0.5f * z : 0.f);
    }
    default: return 1.f;
  }
}

}  // namespace hb
