// Pointwise activation kernels: HardMish and NLReLU, forward and backward.
//
// Reference semantics (holocron/nn/functional.py:30-56 of frgfm/Holocron):
//   hard_mish(x) = 0.5 * x * clamp(x + 2, 0, 2)
//   nl_relu(x)   = log(1 + beta * relu(x))
// Backward semantics are those autograd derives from the reference compositions
// (SURVEY.md §10.3): inclusive clamp mask for hard_mish, relu'(0) = 0 for nl_relu.
//
// All kernels are single HBM passes: 128-bit loads/stores, 4 independent vectors in flight
// per thread, grid capped at a multiple of the SM count with a grid-stride loop.
#include "common.cuh"

namespace {

using namespace hb;

struct HardMishFwd {
  __device__ __forceinline__ float operator()(float x) const {
    // 0.5 * x * clamp(x + 2, 0, 2): same association as the reference ((0.5*x) * clamp)
    float c = fminf(fmaxf(x + 2.0f, 0.0f), 2.0f);
    return (0.5f * x) * c;
  }
};
struct HardMishBwd {
  // d/dx [0.5 x clamp(x+2,0,2)] = 0.5*clamp(x+2,0,2) + 0.5*x*[0 <= x+2 <= 2]. As in autograd, the clamp's mask selects
  // (x = +-inf gives dy or 0, not inf * 0) and a NaN input propagates.
  __device__ __forceinline__ float operator()(float x, float dy) const {
    const float t = x + 2.0f;
    const float c = hb::clamp_nan(t, 0.0f, 2.0f);
    const float inner = (t >= 0.0f && t <= 2.0f) ? 0.5f * x : 0.0f;
    return dy * (0.5f * c + inner);
  }
};
// kFast (16-bit storage types): MUFU log / reciprocal. The argument is >= 1, where __logf is within 2^-21.4 absolute
// error, 2^7 times finer than the bf16 / fp16 rounding of the result; IEEE logf makes the forward pass instruction bound.
// fp32 tensors keep logf and IEEE division.
template <bool kFast>
struct NLReluFwd {
  float beta;
  __device__ __forceinline__ float operator()(float x) const {
    const float a = 1.0f + beta * hb::relu_nan(x);
    return kFast ? __logf(a) : logf(a);
  }
};
template <bool kFast>
struct NLReluBwd {
  float beta;
  __device__ __forceinline__ float operator()(float x, float dy) const {
    if (x <= 0.0f) return 0.0f;  // relu'(0) = 0; a NaN input propagates, as through autograd's threshold_backward
    return kFast ? dy * __fdividef(beta, 1.0f + beta * x) : dy * (beta / (1.0f + beta * x));
  }
};
struct NLReluBwdFromOut {
  // y = log(1 + beta*relu(x))  =>  for y > 0: dy/dx = beta * exp(-y); else 0
  float beta;
  __device__ __forceinline__ float operator()(float y, float dy) const {
    return y <= 0.0f ? 0.0f : dy * (beta * expf(-y));  // NaN propagates as in the out-of-place gradient
  }
};

constexpr int kThreads = 256;
constexpr int kUnroll = 4;

template <typename T, typename Op>
__global__ void __launch_bounds__(kThreads) unary_kernel(const T* x, T* y, size_t n, Op op,
                                                          bool vec_ok) {
  constexpr int V = Vec16<T>::N;
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t nthreads = (size_t)gridDim.x * blockDim.x;
  size_t nvec = vec_ok ? n / V : 0;
  // main body: kUnroll vectors per thread per trip, loads issued before any use
  size_t i = tid;
  for (; i + (kUnroll - 1) * nthreads < nvec; i += kUnroll * nthreads) {
    Vec16<T> in[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) in[u] = ld16_stream(x + (i + u * nthreads) * V);
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      Vec16<T> o;
#pragma unroll
      for (int k = 0; k < V; ++k) o.v[k] = from_f<T>(op(to_f(in[u].v[k])));
      st16(y + (i + u * nthreads) * V, o);
    }
  }
  for (; i < nvec; i += nthreads) {
    Vec16<T> a = ld16_stream(x + i * V), o;
#pragma unroll
    for (int k = 0; k < V; ++k) o.v[k] = from_f<T>(op(to_f(a.v[k])));
    st16(y + i * V, o);
  }
  // scalar tail (or everything when the pointers are not 16B aligned)
  for (size_t j = nvec * V + tid; j < n; j += nthreads) y[j] = from_f<T>(op(to_f(x[j])));
}

template <typename T, typename Op>
__global__ void __launch_bounds__(kThreads) binary_kernel(const T* __restrict__ a, const T* __restrict__ b,
                                                           T* __restrict__ y, size_t n, Op op, bool vec_ok) {
  constexpr int V = Vec16<T>::N;
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t nthreads = (size_t)gridDim.x * blockDim.x;
  size_t nvec = vec_ok ? n / V : 0;
  size_t i = tid;
  constexpr int U = 2;
  for (; i + (U - 1) * nthreads < nvec; i += U * nthreads) {
    Vec16<T> va[U], vb[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      va[u] = ld16_stream(a + (i + u * nthreads) * V);
      vb[u] = ld16_stream(b + (i + u * nthreads) * V);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      Vec16<T> o;
#pragma unroll
      for (int k = 0; k < V; ++k) o.v[k] = from_f<T>(op(to_f(va[u].v[k]), to_f(vb[u].v[k])));
      st16(y + (i + u * nthreads) * V, o);
    }
  }
  for (; i < nvec; i += nthreads) {
    Vec16<T> va = ld16_stream(a + i * V), vb = ld16_stream(b + i * V), o;
#pragma unroll
    for (int k = 0; k < V; ++k) o.v[k] = from_f<T>(op(to_f(va.v[k]), to_f(vb.v[k])));
    st16(y + i * V, o);
  }
  for (size_t j = nvec * V + tid; j < n; j += nthreads) y[j] = from_f<T>(op(to_f(a[j]), to_f(b[j])));
}

template <typename T, typename Op>
int launch_unary(const void* x, void* y, size_t n, Op op, cudaStream_t s) {
  if (n == 0) return 0;
  constexpr int V = Vec16<T>::N;
  bool vec_ok = aligned16(x) && aligned16(y);
  int grid = stream_grid(n, kThreads * V * kUnroll);
  unary_kernel<T, Op><<<grid, kThreads, 0, s>>>((const T*)x, (T*)y, n, op, vec_ok);
  HB_LAUNCH_CHECK();
  return 0;
}
template <typename T, typename Op>
int launch_binary(const void* a, const void* b, void* y, size_t n, Op op, cudaStream_t s) {
  if (n == 0) return 0;
  constexpr int V = Vec16<T>::N;
  bool vec_ok = aligned16(a) && aligned16(b) && aligned16(y);
  int grid = stream_grid(n, kThreads * V * 2);
  binary_kernel<T, Op><<<grid, kThreads, 0, s>>>((const T*)a, (const T*)b, (T*)y, n, op, vec_ok);
  HB_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" {

int hb_hard_mish_fwd(const void* x, void* y, size_t n, int dtype, void* stream) {
  return dispatch_dtype(dtype, [&](auto type) {
    return launch_unary<typename decltype(type)::type>(x, y, n, HardMishFwd{}, (cudaStream_t)stream);
  });
}
int hb_hard_mish_bwd(const void* x, const void* dy, void* dx, size_t n, int dtype, void* stream) {
  return dispatch_dtype(dtype, [&](auto type) {
    return launch_binary<typename decltype(type)::type>(x, dy, dx, n, HardMishBwd{}, (cudaStream_t)stream);
  });
}
int hb_nl_relu_fwd(const void* x, void* y, size_t n, float beta, int dtype, void* stream) {
  return dispatch_dtype(dtype, [&](auto type) {
    using T = typename decltype(type)::type;
    return launch_unary<T>(x, y, n, NLReluFwd<(sizeof(T) < 4)>{beta}, (cudaStream_t)stream);
  });
}
int hb_nl_relu_bwd(const void* x, const void* dy, void* dx, size_t n, float beta, int dtype, void* stream) {
  return dispatch_dtype(dtype, [&](auto type) {
    using T = typename decltype(type)::type;
    return launch_binary<T>(x, dy, dx, n, NLReluBwd<(sizeof(T) < 4)>{beta}, (cudaStream_t)stream);
  });
}
int hb_nl_relu_bwd_from_out(const void* y, const void* dy, void* dx, size_t n, float beta, int dtype, void* stream) {
  return dispatch_dtype(dtype, [&](auto type) {
    return launch_binary<typename decltype(type)::type>(y, dy, dx, n, NLReluBwdFromOut{beta}, (cudaStream_t)stream);
  });
}

}  // extern "C"
