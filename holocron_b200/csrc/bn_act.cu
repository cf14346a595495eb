// Training-mode BatchNorm + branch-sum + activation, fused for NHWC bf16 activations.
//
// The unit being fused is the reference's "conv -> BatchNorm2d -> act" sequence
// (holocron/models/utils.py:28-86 conv_sequence) and the RepVGG block
//   out = act( BN3(conv3x3(x)) + BN1(conv1x1(x)) [+ BNid(x)] )        (models/classification/repvgg.py:71-73)
// generalised to B <= 3 normalised branches u_b of identical shape [M, C] plus an optional un-normalised
// residual. The reference runs one cuDNN/ATen kernel per BN, add and activation (>= 8 HBM passes per
// RepBlock); here the whole thing is
//   stats      : per-channel sum / sum-of-squares PARTIALS, normally produced by whoever wrote the tensor (the epilogue of
//                the tensor-core convolution, conv_fprop.cu / conv_rows.cu, or the forward pass below for a block's own
//                output); bn_stats_partials_kernel is the stand-alone pass for tensors that come without partials
//   finalize   : C-sized: fixed-order fp64 sum of the partials (deterministic: no floating-point atomics anywhere),
//                mean, rstd, scale = gamma*rstd, shift = beta - mean*scale, running-stat update
//   forward    : one pass: out = act(sum_b (scale_b * u_b + shift_b) + residual)
//   bwd reduce : one pass: sum(dz), sum(dz * xhat_b)    with dz = dOut * act'(z), z recomputed (not stored)
//   bwd apply  : one pass: du_b = scale_b * (dz - mean(dz) - xhat_b * mean(dz*xhat_b)), dresidual = dz
// Every thread owns 8 consecutive channels (one 128-bit bf16 vector) of a row; rows are walked with a stride
// that keeps the thread's channel group fixed, so per-channel parameters live in registers.
#include <cstdio>
#include <cstdlib>
#include <type_traits>
#include <utility>
#include "common.cuh"
#include "act.cuh"
#include "slab.cuh"

namespace {

using namespace hb;

constexpr int kThreads = kSlabThreads;
constexpr int kMaxBranches = 3;

struct Branches {
  const __nv_bfloat16* u[kMaxBranches];
  int n;
};

// (sum, sum of squares) partials of this block's rows, from the [2][kThreads * 8] lane values in red: parts[blockIdx.x][c]
// as one float2 per channel ([slots][C][2], the layout hb_bn_finalize reads)
__device__ __forceinline__ void fold_stat_partials(const SlabGeo& g, const float* red, int C, float* parts) {
  fold_row_lanes<double, 2>(g, red, [&](int c, const double (&a)[2]) {
    *reinterpret_cast<float2*>(parts + ((size_t)blockIdx.x * C + c) * 2) = make_float2((float)a[0], (float)a[1]);
  });
}

// ---------------------------------------------------------------------------------------------------
// stand-alone statistics pass: parts[blockIdx.x][c] = (sum, sum of squares) of this block's rows of u [M, C]
// grid = (row blocks = slots, channel slabs)
__global__ void __launch_bounds__(kThreads) bn_stats_partials_kernel(const __nv_bfloat16* __restrict__ u, int M, int C,
                                                                     SlabGeo g, float* __restrict__ parts) {
  __shared__ float red[2][kThreads * 8];
  const auto [tx, ty, cg, active] = g.thread();
  float s[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { s[j] = 0.f; q[j] = 0.f; }
  if (active) {
    const size_t row_stride = (size_t)gridDim.x * g.rows_t;
    size_t m = (size_t)blockIdx.x * g.rows_t + ty;
    // two rows in flight per trip
    for (; m + row_stride < (size_t)M; m += 2 * row_stride) {
      float a[8], b[8];
      unpack8(ld16_stream(u + m * C + cg * 8), a);
      unpack8(ld16_stream(u + (m + row_stride) * C + cg * 8), b);
#pragma unroll
      for (int j = 0; j < 8; ++j) { s[j] += a[j] + b[j]; q[j] += a[j] * a[j] + b[j] * b[j]; }
    }
    if (m < (size_t)M) {
      float a[8];
      unpack8(ld16_stream(u + m * C + cg * 8), a);
#pragma unroll
      for (int j = 0; j < 8; ++j) { s[j] += a[j]; q[j] += a[j] * a[j]; }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) { red[0][threadIdx.x * 8 + j] = s[j]; red[1][threadIdx.x * 8 + j] = q[j]; }
  __syncthreads();
  fold_stat_partials(g, &red[0][0], C, parts);
}

// ---------------------------------------------------------------------------------------------------
// finalize: per branch b and channel c
struct FinalizeParams {
  const float* parts[kMaxBranches];   // [slots_b][C][2] (sum, sum of squares) partials
  int slots[kMaxBranches];
  const float* gamma[kMaxBranches];
  const float* beta[kMaxBranches];
  float* running_mean[kMaxBranches];  // may be null
  float* running_var[kMaxBranches];
  long long* num_batches_tracked[kMaxBranches];  // int64 scalar per branch, may be null
  float* mean;   // [B][C] out
  float* rstd;   // [B][C] out
  float* scale;  // [B][C] out
  float* shift;  // [B][C] out
  int B, C, M;
  int C_logical;  // channels >= C_logical are padding: scale = shift = 0, no parameter / running-stat access
  float eps, momentum;
  double* sums;   // [B][C][2] (sum, sum of squares) + the row count: written by bn_partials_sums_kernel, read by
                  // bn_finalize_sums_kernel (a synchronised BatchNorm all-reduces it in between)
};
// block = 8 channels (threadIdx.x: one 64-byte run of the [slot][C][2] partials) x 32 slot lanes (threadIdx.y). A lane adds
// slots L, L + 32, ... with four independent loads in flight, the 32 lane sums are then combined 8-by-8 in lane order: a
// fixed summation order (run-to-run identical) whose dependent-load chain is slots / 128 long. (32 channels x 8 lanes: slots /
// 8 dependent L2 round trips and C / 32 blocks - two blocks for a 48-channel layer - is latency bound.)
constexpr int kFinCh = 8, kFinLanes = 32;

// The fold of both finalize kernels: NS sums of n slots (of which the first `live` are used), read by load(k, v) as the NS
// values of slot k. Returns the totals in the threads with threadIdx.y == 0; every thread must call it (it synchronises).
template <int NS, typename Load>
__device__ __forceinline__ void fold_slots(bool has_slots, int n, int live, Load load, double (&tot)[NS]) {
  __shared__ double red[NS][kFinLanes][kFinCh];
  double acc[NS];
#pragma unroll
  for (int i = 0; i < NS; ++i) acc[i] = 0.0;
  if (has_slots) {
    int k = threadIdx.y;
    for (; k + 3 * kFinLanes < n; k += 4 * kFinLanes) {
      double v[4][NS];
#pragma unroll
      for (int u = 0; u < 4; ++u) load(k + u * kFinLanes, v[u]);
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int i = 0; i < NS; ++i)
          if (i < live) acc[i] += v[u][i];
    }
    for (; k < n; k += kFinLanes) {
      double v[NS];
      load(k, v);
#pragma unroll
      for (int i = 0; i < NS; ++i)
        if (i < live) acc[i] += v[i];
    }
  }
#pragma unroll
  for (int i = 0; i < NS; ++i) red[i][threadIdx.y][threadIdx.x] = acc[i];
  __syncthreads();
  if (threadIdx.y < 4) {
#pragma unroll
    for (int i = 0; i < NS; ++i) {
      double t = 0.0;
#pragma unroll
      for (int j = 0; j < 8; ++j) t += red[i][threadIdx.y * 8 + j][threadIdx.x];
      acc[i] = t;
    }
  }
  __syncthreads();
  if (threadIdx.y < 4) {
#pragma unroll
    for (int i = 0; i < NS; ++i) red[i][threadIdx.y][threadIdx.x] = acc[i];
  }
  __syncthreads();
  if (threadIdx.y != 0) return;
#pragma unroll
  for (int i = 0; i < NS; ++i) {
    double t = 0.0;
#pragma unroll
    for (int j = 0; j < 4; ++j) t += red[i][j][threadIdx.x];
    tot[i] = t;
  }
}

// Branch b, channel c of the finalisation from the fp64 (sum, sum of squares) s, q over n rows: mean / rstd / scale / shift,
// the running statistics (unbiased variance over n) and num_batches_tracked. n is the local row count (hb_bn_finalize) or
// the count summed over the ranks of a synchronised BatchNorm (hb_bn_finalize_sums); for an integer n both read the same.
__device__ __forceinline__ void finalize_channel(const FinalizeParams& p, int b, int c, double s, double q, double n) {
  const size_t o = (size_t)b * p.C + c;
  if (c >= p.C_logical) {
    p.mean[o] = 0.f; p.rstd[o] = 0.f; p.scale[o] = 0.f; p.shift[o] = 0.f;
    return;
  }
  const double mean = s / n;
  double var = q / n - mean * mean;
  if (var < 0) var = 0;
  const float rstd = (float)(1.0 / sqrt(var + (double)p.eps));
  const float g = p.gamma[b] ? p.gamma[b][c] : 1.f;
  const float be = p.beta[b] ? p.beta[b][c] : 0.f;
  const float sc = g * rstd;
  p.mean[o] = (float)mean;
  p.rstd[o] = rstd;
  p.scale[o] = sc;
  p.shift[o] = be - (float)mean * sc;
  if (c == 0 && p.num_batches_tracked[b]) *p.num_batches_tracked[b] += 1;
  if (p.running_mean[b]) {
    const double unbiased = n > 1.0 ? var * (n / (n - 1.0)) : var;
    p.running_mean[b][c] = (1.f - p.momentum) * p.running_mean[b][c] + p.momentum * (float)mean;
    p.running_var[b][c] = (1.f - p.momentum) * p.running_var[b][c] + p.momentum * (float)unbiased;
  }
}

// (sum, sum of squares) of branch b, channel c over the branch's partial slots, in the fixed order of fold_slots; returned in
// the threads with threadIdx.y == 0 (every thread of the block must call it)
__device__ __forceinline__ void fold_partials(const FinalizeParams& p, int b, int c, double (&tot)[2]) {
  const float* pp = p.parts[b] + (size_t)c * 2;
  const size_t row = (size_t)p.C * 2;
  fold_slots<2>(c < p.C_logical, p.slots[b], 2, [&](int k, double (&v)[2]) {
    const float2 f = *reinterpret_cast<const float2*>(pp + (size_t)k * row);
    v[0] = (double)f.x; v[1] = (double)f.y;
  }, tot);
}

__global__ void __launch_bounds__(kFinCh * kFinLanes) bn_finalize_kernel(FinalizeParams p) {
  const int c = blockIdx.x * kFinCh + threadIdx.x;
  const int b = blockIdx.y;
  double tot[2];
  fold_partials(p, b, c, tot);
  if (threadIdx.y != 0 || c >= p.C) return;
  finalize_channel(p, b, c, tot[0], tot[1], (double)p.M);
}

// synchronised BatchNorm, step 1: the same fixed-order fold, written out as sums[b][c] = (sum, sum of squares) and
// sums[B][0][0] = M (a double, so that the count adds up over ranks with the sums)
__global__ void __launch_bounds__(kFinCh * kFinLanes) bn_partials_sums_kernel(FinalizeParams p) {
  const int c = blockIdx.x * kFinCh + threadIdx.x;
  const int b = blockIdx.y;
  double tot[2];
  fold_partials(p, b, c, tot);
  if (threadIdx.y != 0 || c >= p.C) return;
  const size_t o = ((size_t)b * p.C + c) * 2;
  p.sums[o] = tot[0];
  p.sums[o + 1] = tot[1];
  if (b == 0 && c == 0) p.sums[(size_t)p.B * p.C * 2] = (double)p.M;
}

// synchronised BatchNorm, step 2: finalisation from the all-reduced sums and count
__global__ void bn_finalize_sums_kernel(FinalizeParams p) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (c >= p.C) return;
  const size_t o = ((size_t)b * p.C + c) * 2;
  finalize_channel(p, b, c, p.sums[o], p.sums[o + 1], p.sums[(size_t)p.B * p.C * 2]);
}

// eval-mode affine from running statistics: scale = gamma / sqrt(var + eps), shift = beta - mean * scale
__global__ void bn_eval_affine_kernel(const float* gamma, const float* beta, const float* rmean, const float* rvar,
                                      float eps, int C, int C_logical, float* scale, float* shift, float* mean,
                                      float* rstd) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (c >= C_logical) {
    scale[c] = 0.f; shift[c] = 0.f;
    if (mean) mean[c] = 0.f;
    if (rstd) rstd[c] = 0.f;
    return;
  }
  const float r = 1.f / sqrtf(rvar[c] + eps);
  const float sc = (gamma ? gamma[c] : 1.f) * r;
  scale[c] = sc;
  shift[c] = (beta ? beta[c] : 0.f) - rmean[c] * sc;
  if (mean) mean[c] = rmean[c];
  if (rstd) rstd[c] = r;
}

// ---------------------------------------------------------------------------------------------------
// forward: out = act(sum_b scale_b*u_b + shift_b (+ residual))
struct FwdParams {
  Branches br;
  const float* scale;  // [B][C]
  const float* shift;  // [B][C]
  const __nv_bfloat16* residual;
  __nv_bfloat16* out;
  int M, C, act;
  float slope;
  int res_after;  // 1: out = act(z) + residual (ResNet-style shortcut after the activation); 0: act(z + residual)
  float* out_stats;  // optional [gridDim.x][C][2]: (sum, sum of squares) partials of the bf16 OUTPUT - the statistics the
                     // identity-branch BatchNorm of the NEXT RepVGG block needs, produced while the data is in registers
};
using RawVec = Vec16<__nv_bfloat16>;

// 8 floats of a per-channel constant in shared memory, as two float4
__device__ __forceinline__ void lds8(const float* p, float* f) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

// ---- per-thread cp.async ring ---------------------------------------------------------------------
// Every thread streams ITS OWN 16-byte vectors (one per input tensor and row) global -> shared with cp.async, kDepth rows
// ahead of the row it is computing on; nothing else reads those slots, so the ring needs no barrier at all. This puts
// kDepth * (#inputs) * 16 B per thread in flight without holding them in registers: the register-staged version of these
// kernels had far fewer bytes per SM in flight than the HBM bandwidth x loaded latency product and stalled on long
// scoreboard waits.
// rows in flight per thread as a function of the number of streamed tensors NT: what matters is BYTES in flight per SM
// (depth * NT * 16 B * 256 threads * resident blocks). With depth 3 the single-branch units (ReXNet / Darknet / UNet3+ /
// YOLOv4: one input tensor) keep too few bytes in flight with depth 3; deeper rings for fewer tensors.
// depth + 1 slots: keep the slot count a power of two (the slot index is k % slots on a 64-bit row counter)
__host__ __device__ constexpr int ring_depth(int nt) { return nt <= 2 ? 7 : 3; }

__device__ __forceinline__ void cp_async16(uint32_t saddr, const void* g) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(saddr), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ RawVec lds16(uint32_t saddr) {
  RawVec r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.raw.x), "=r"(r.raw.y), "=r"(r.raw.z), "=r"(r.raw.w) : "r"(saddr));
  return r;
}
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Walks the rows m = m0, m0 + stride, ... < M of one thread. NT input tensors; src[t] is tensor t's base pointer (set by
// the kernel after init; a null source is not streamed).
template <int NT>
struct RowRing {
  static constexpr int kDepth = ring_depth(NT);
  static constexpr int kSlots = kDepth + 1;   // the slot refilled at step k is the one consumed at step k-1
  uint32_t base;       // shared address of this thread's slot 0 / tensor 0
  size_t m0, stride, M;
  size_t col_off;      // element offset of the thread's 8 channels inside a row
  int C;
  const __nv_bfloat16* src[NT > 0 ? NT : 1];
  __device__ __forceinline__ void init(uint8_t* smem, size_t m0_, size_t stride_, int M_, int C_, size_t col_off_) {
    base = smem_addr(smem) + threadIdx.x * 16;
    m0 = m0_; stride = stride_; M = (size_t)M_; col_off = col_off_; C = C_;
  }
  // slot s, tensor t of this thread
  __device__ __forceinline__ uint32_t addr(int s, int t) const { return base + (uint32_t)((s * NT + t) * kThreads * 16); }
  __device__ __forceinline__ bool valid(size_t k) const { return m0 + k * stride < M; }
  __device__ __forceinline__ size_t off(size_t k) const { return (m0 + k * stride) * C + col_off; }
  __device__ __forceinline__ void issue(size_t k) const {
    if (valid(k)) {
      const int s = (int)(k % kSlots);
      const size_t o = off(k);
#pragma unroll
      for (int t = 0; t < NT; ++t)
        if (src[t]) cp_async16(addr(s, t), src[t] + o);
    }
    cp_async_commit();   // always: keeps the group count uniform
  }
  __device__ __forceinline__ void prologue() const {
#pragma unroll
    for (int k = 0; k < kDepth; ++k) issue(k);
  }
  // row k has landed
  __device__ __forceinline__ void wait() const { cp_async_wait<kDepth - 1>(); }
};

// forward: out = act(sum_b scale_b*u_b + shift_b (+ residual))
// kStats: also accumulate the output statistics (separate instantiation: the plain kernel keeps its register budget; with
// the 16 extra accumulators the 3-branch kernel would drop from 3 to 2 resident blocks per SM, so the statistics variant is
// compiled for 3 blocks explicitly)
template <int NB, bool kStats>
__global__ void __launch_bounds__(kThreads, 3) bn_act_fwd_kernel(FwdParams p, SlabGeo g) {
  extern __shared__ __align__(16) uint8_t ring_smem[];
  const auto [tx, ty, cg, active] = g.thread();
  float os[8], oq[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { os[j] = 0.f; oq[j] = 0.f; }
  // folded per-channel constants of this block's channel slab live in shared memory (read as float4 pairs per row): with
  // them in registers the statistics variant of the 3-branch kernel spilled inside the streaming loop
  __shared__ __align__(16) float k_sc[kMaxBranches][256];
  __shared__ __align__(16) float k_sh[256];
  {
    const int nch = g.cg_t * 8;
    for (int ch = threadIdx.x; ch < nch; ch += kThreads) {
      const int c = blockIdx.y * nch + ch;
      float shv = 0.f;
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        k_sc[b][ch] = c < p.C ? p.scale[(size_t)b * p.C + c] : 0.f;
        shv += c < p.C ? p.shift[(size_t)b * p.C + c] : 0.f;
      }
      k_sh[ch] = shv;
    }
    __syncthreads();
  }
  if (!active && !kStats) return;
  if (active) {
    const bool has_res = p.residual != nullptr;
    RowRing<NB + 1> ring;
    ring.init(ring_smem, (size_t)blockIdx.x * g.rows_t + ty, (size_t)gridDim.x * g.rows_t, p.M, p.C, (size_t)cg * 8);
#pragma unroll
    for (int b = 0; b < NB; ++b) ring.src[b] = p.br.u[b];
    ring.src[NB] = p.residual;
    ring.prologue();
    for (size_t k = 0; ring.valid(k); ++k) {
      ring.wait();
      const int s = (int)(k % RowRing<NB + 1>::kSlots);
      RawVec u[NB > 0 ? NB : 1], r;
#pragma unroll
      for (int b = 0; b < NB; ++b) u[b] = lds16(ring.addr(s, b));
      if (has_res) r = lds16(ring.addr(s, NB));
      ring.issue(k + RowRing<NB + 1>::kDepth);
      float z[8];
      lds8(&k_sh[tx * 8], z);
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        float f[8], sc[8];
        lds8(&k_sc[b][tx * 8], sc);
        unpack8(u[b], f);
#pragma unroll
        for (int j = 0; j < 8; ++j) z[j] = fmaf(sc[j], f[j], z[j]);
      }
      float rr[8];
      if (has_res) unpack8(r, rr);
      if (has_res && !p.res_after) {
        if (p.act == ACT_FRELU) {
#pragma unroll
          for (int j = 0; j < 8; ++j) z[j] = max_nan(z[j], rr[j]);
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) z[j] += rr[j];
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) z[j] = act_fwd(p.act, z[j], p.slope);
      if (has_res && p.res_after) {
#pragma unroll
        for (int j = 0; j < 8; ++j) z[j] += rr[j];
      }
      Vec16<__nv_bfloat16> ov;
#pragma unroll
      for (int j = 0; j < 8; ++j) ov.v[j] = __float2bfloat16_rn(z[j]);
      st16(p.out + ring.off(k), ov);
      if (kStats) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float f = __bfloat162float(ov.v[j]);   // statistics of what the consumer will read
          os[j] += f; oq[j] = fmaf(f, f, oq[j]);
        }
      }
    }
  }
  if (!kStats) return;
  // block partial of the output statistics: the ring memory is free now (every cp.async group has been waited for)
  cp_async_wait<0>();
  __syncthreads();
  float* red = reinterpret_cast<float*>(ring_smem);   // [2][kThreads * 8] floats = 16 KB <= smallest ring
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    red[threadIdx.x * 8 + j] = active ? os[j] : 0.f;
    red[kThreads * 8 + threadIdx.x * 8 + j] = active ? oq[j] : 0.f;
  }
  __syncthreads();
  fold_stat_partials(g, red, p.C, p.out_stats);
}

// ---------------------------------------------------------------------------------------------------
// backward
struct BwdParams {
  Branches br;
  const __nv_bfloat16* dout;
  const __nv_bfloat16* residual;
  const float* scale;  // [B][C]
  const float* shift;
  const float* mean;
  const float* rstd;
  double* sums;        // [1 + B][C]: sum dz, sum dz*u_b (final, written by bn_bwd_finalize_kernel)
  double* part;        // [row blocks][1 + B][C]: per-block partials of the above (pass 1), summed in a fixed order
  const double* count; // row count the sums are over (device scalar: summed over the ranks of a synchronised BatchNorm);
                       // null: M
  __nv_bfloat16* du[kMaxBranches];
  __nv_bfloat16* dres;  // may be null
  int M, C, act;
  float slope;
  int train;  // 1: batch statistics (full BN backward); 0: running statistics (du = scale * dz)
  int res_after;
};

// Per-channel constants of the block's channel slab in shared memory, read as float4 pairs (8 channels per thread).
//   z    = sum_b scale_b * u_b + shift
//   du_b = scale_b * (dz - mean(dz) - xhat_b * mean(dz * xhat_b))  =  scale_b * dz + cu_b * u_b + c0_b
// with cu_b = -scale_b * rstd_b * mdzx_b, c0_b = -scale_b * mdz - cu_b * mean_b and
// mdzx_b = mean(dz * xhat_b) = rstd_b * (sum(dz * u_b) / M - mean_b * mdz) from the first pass' sums.
struct SlabConsts {
  float scale[kMaxBranches][256];
  float cu[kMaxBranches][256];
  float c0[kMaxBranches][256];
  float shift[256];   // sum over branches
};

template <int NB>
__device__ __forceinline__ void load_slab_consts(SlabConsts& k, const BwdParams& p, const SlabGeo& g, bool with_means) {
  const int nch = g.cg_t * 8;
  const double invM = 1.0 / (p.count ? *p.count : (double)p.M);
  for (int ch = threadIdx.x; ch < nch; ch += kThreads) {
    const int c = blockIdx.y * nch + ch;
    const bool ok = c < p.C;
    float sh = 0.f;
    const double mdz = (with_means && p.train && ok) ? p.sums[c] * invM : 0.0;
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      const size_t o = (size_t)b * p.C + c;
      const float sc = ok ? p.scale[o] : 0.f;
      k.scale[b][ch] = sc;
      sh += ok ? p.shift[o] : 0.f;
      float cu = 0.f, c0 = 0.f;
      if (with_means && p.train && ok) {
        const double mean = (double)p.mean[o], rstd = (double)p.rstd[o];
        const double mdzx = rstd * (p.sums[(size_t)(1 + b) * p.C + c] * invM - mean * mdz);
        const double cud = -(double)sc * rstd * mdzx;
        cu = (float)cud;
        c0 = (float)(-(double)sc * mdz - cud * mean);
      }
      k.cu[b][ch] = cu;
      k.c0[b][ch] = c0;
    }
    k.shift[ch] = sh;
  }
  __syncthreads();
}

// dz = d out / d z (z = normalised branch sum [+ residual]); dr = gradient reaching the residual input
template <int NB>
__device__ __forceinline__ void recompute_dz(const BwdParams& p, const SlabConsts& k, int ch0, const RawVec* uv,
                                             const RawVec& rv, const RawVec& dv, float (*u)[8], float* dz, float* dr) {
  float z[8];
  lds8(&k.shift[ch0], z);
#pragma unroll
  for (int b = 0; b < NB; ++b) {
    float sc[8];
    lds8(&k.scale[b][ch0], sc);
    unpack8(uv[b], u[b]);
#pragma unroll
    for (int j = 0; j < 8; ++j) z[j] = fmaf(sc[j], u[b][j], z[j]);
  }
  float d[8];
  unpack8(dv, d);
  if (p.residual && p.res_after) {
#pragma unroll
    for (int j = 0; j < 8; ++j) { dz[j] = d[j] * act_grad(p.act, z[j], p.slope); dr[j] = d[j]; }
    return;
  }
  if (p.residual) {
    float r[8];
    unpack8(rv, r);
    if (p.act == ACT_FRELU) {
      // binary max: the gradient goes to the larger argument, ties are split evenly (PyTorch semantics)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float gate = z[j] > r[j] ? 1.f : (z[j] == r[j] ? 0.5f : 0.f);
        dz[j] = d[j] * gate;
        dr[j] = d[j] - dz[j];
      }
      return;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) z[j] += r[j];
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) { dz[j] = d[j] * act_grad(p.act, z[j], p.slope); dr[j] = dz[j]; }
}

template <int NB>
__device__ __forceinline__ void init_bwd_ring(RowRing<NB + 2>& ring, const BwdParams& p, const SlabGeo& g, uint8_t* ring_smem,
                                              int ty, int cg) {
  ring.init(ring_smem, (size_t)blockIdx.x * g.rows_t + ty, (size_t)gridDim.x * g.rows_t, p.M, p.C, (size_t)cg * 8);
#pragma unroll
  for (int b = 0; b < NB; ++b) ring.src[b] = p.br.u[b];
  ring.src[NB] = (p.residual && !p.res_after) ? p.residual : nullptr;   // its value only matters inside act()
  ring.src[NB + 1] = p.dout;
}

// pass 1: part[blk][0][c] = sum_m dz, part[blk][1+b][c] = sum_m dz * u_b over the rows of this block (no atomics)
template <int NB>
__global__ void __launch_bounds__(kThreads, 2) bn_act_bwd_reduce_kernel(BwdParams p, SlabGeo g) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  SlabConsts& k = *reinterpret_cast<SlabConsts*>(dyn_smem);
  float* red = reinterpret_cast<float*>(dyn_smem + sizeof(SlabConsts));   // [kThreads * 8]
  uint8_t* ring_smem = dyn_smem + sizeof(SlabConsts) + kThreads * 8 * sizeof(float);
  load_slab_consts<NB>(k, p, g, false);
  const auto [tx, ty, cg, active] = g.thread();
  float acc[1 + NB][8];
#pragma unroll
  for (int i = 0; i < 1 + NB; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  if (active) {
    RowRing<NB + 2> ring;
    init_bwd_ring<NB>(ring, p, g, ring_smem, ty, cg);
    ring.prologue();
    for (size_t kk = 0; ring.valid(kk); ++kk) {
      ring.wait();
      const int s = (int)(kk % RowRing<NB + 2>::kSlots);
      RawVec uv[NB > 0 ? NB : 1], rv, dv;
#pragma unroll
      for (int b = 0; b < NB; ++b) uv[b] = lds16(ring.addr(s, b));
      if (ring.src[NB]) rv = lds16(ring.addr(s, NB));
      dv = lds16(ring.addr(s, NB + 1));
      ring.issue(kk + RowRing<NB + 2>::kDepth);
      float u[NB > 0 ? NB : 1][8], dz[8], dr[8];
      recompute_dz<NB>(p, k, tx * 8, uv, rv, dv, u, dz, dr);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[0][j] += dz[j];
#pragma unroll
      for (int b = 0; b < NB; ++b) {
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[1 + b][j] = fmaf(dz[j], u[b][j], acc[1 + b][j]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 1 + NB; ++i) {
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) red[threadIdx.x * 8 + j] = acc[i][j];
    __syncthreads();
    fold_row_lanes<double, 1>(g, red, [&](int c, const double (&a)[1]) {
      p.part[((size_t)blockIdx.x * (1 + NB) + i) * p.C + c] = a[0];
    });
  }
}

// pass 2: du_b = scale_b * dz + cu_b * u_b + c0_b, dres = dr
template <int NB>
__global__ void __launch_bounds__(kThreads, 2) bn_act_bwd_apply_kernel(BwdParams p, SlabGeo g) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  SlabConsts& k = *reinterpret_cast<SlabConsts*>(dyn_smem);
  uint8_t* ring_smem = dyn_smem + sizeof(SlabConsts);
  load_slab_consts<NB>(k, p, g, true);
  const auto [tx, ty, cg, active] = g.thread();
  if (!active) return;
  RowRing<NB + 2> ring;
  init_bwd_ring<NB>(ring, p, g, ring_smem, ty, cg);
  ring.prologue();
  for (size_t kk = 0; ring.valid(kk); ++kk) {
    ring.wait();
    const int s = (int)(kk % RowRing<NB + 2>::kSlots);
    RawVec uv[NB > 0 ? NB : 1], rv, dv;
#pragma unroll
    for (int b = 0; b < NB; ++b) uv[b] = lds16(ring.addr(s, b));
    if (ring.src[NB]) rv = lds16(ring.addr(s, NB));
    dv = lds16(ring.addr(s, NB + 1));
    ring.issue(kk + RowRing<NB + 2>::kDepth);
    const size_t off = ring.off(kk);
    float u[NB > 0 ? NB : 1][8], dz[8], dr[8];
    recompute_dz<NB>(p, k, tx * 8, uv, rv, dv, u, dz, dr);
    if (p.dres) store8(p.dres + off, dr);
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      if (p.du[b]) {
        float sc[8], cu[8], c0[8], d[8];
        lds8(&k.scale[b][tx * 8], sc);
        lds8(&k.cu[b][tx * 8], cu);
        lds8(&k.c0[b][tx * 8], c0);
#pragma unroll
        for (int j = 0; j < 8; ++j) d[j] = fmaf(sc[j], dz[j], fmaf(cu[j], u[b][j], c0[j]));
        store8(p.du[b] + off, d);
      }
    }
  }
}

// Between the two passes: sums[i][c] = sum over the row blocks of part[blk][i][c] (one warp per channel, fixed order), then
//   dgamma_b = sum dz*xhat_b = rstd_b * (sum dz*u_b - mean_b * sum dz),   dbeta_b = sum dz     (evaluated in fp64)
// written to dgamma/dbeta ([B][C] fp32, optional) and / or ACCUMULATED into the parameters' gradient buffers gacc/bacc
// (`.grad` storage of the BatchNorm weight / bias: what autograd's AccumulateGrad would do with one more kernel each).
struct BwdFinalizeParams {
  const double* part; double* sums; const float* mean; const float* rstd;
  float* dgamma; float* dbeta;
  float* gacc[kMaxBranches]; float* bacc[kMaxBranches];
  int nblocks, B, C, C_logical;
};
// same block shape as bn_finalize_kernel: 8 channels x 32 row-block lanes, four independent rows in flight, fixed order
__global__ void __launch_bounds__(kFinCh * kFinLanes) bn_bwd_finalize_kernel(BwdFinalizeParams p) {
  const int c = blockIdx.x * kFinCh + threadIdx.x;
  const size_t row = (size_t)(1 + p.B) * p.C;
  double tot[1 + kMaxBranches];
  fold_slots<1 + kMaxBranches>(c < p.C, p.nblocks, 1 + p.B, [&](int k, double (&v)[1 + kMaxBranches]) {
#pragma unroll
    for (int i = 0; i <= kMaxBranches; ++i)
      if (i <= p.B) v[i] = p.part[(size_t)k * row + (size_t)i * p.C + c];
  }, tot);
  if (threadIdx.y != 0 || c >= p.C) return;
  for (int i = 0; i <= p.B; ++i) p.sums[(size_t)i * p.C + c] = tot[i];
  for (int b = 0; b < p.B; ++b) {
    const size_t o = (size_t)b * p.C + c;
    const float dg = (float)((double)p.rstd[o] * (tot[1 + b] - (double)p.mean[o] * tot[0]));
    const float db = (float)tot[0];
    if (p.dgamma) p.dgamma[o] = dg;
    if (p.dbeta) p.dbeta[o] = db;
    if (c < p.C_logical) {
      if (p.gacc[b]) p.gacc[b][c] += dg;
      if (p.bacc[b]) p.bacc[b][c] += db;
    }
  }
}

inline int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v ? atoi(v) : dflt;
}

// Resident blocks per SM of one kernel instantiation with SMEM dynamic bytes. The grids are persistent (every block walks
// M / gridDim.x rows), so a grid of 4 blocks per SM of a kernel that only fits 3 runs as one full wave plus a one-third-occupied
// second wave, which streams markedly slower than a grid of exactly the resident blocks.
template <typename K>
inline int resident_blocks(K kernel, size_t smem) {
  int n = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, kThreads, smem) != cudaSuccess || n < 1) n = 1;
  return n;
}

// One kernel instantiation, ready to launch with SMEM dynamic bytes, and its resident blocks per SM (0: its dynamic
// shared-memory limit could not be raised). Both are set up on the first call only. The cache is keyed on the kernel pointer,
// not its type: every bn_act_fwd_kernel<NB, kStats> has the same function type, and one of them must not use another's count.
template <auto Kernel>
std::pair<decltype(Kernel), int> instance(size_t smem) {
  static int occ = 0;
  if (!occ) {
    if (cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess) return {Kernel, 0};
    occ = resident_blocks(Kernel, smem);
  }
  return {Kernel, occ};
}

// pick(std::integral_constant<int, NB>{}) for NB = B normalised branches (0 .. kMaxBranches, checked by the entry points)
template <typename F>
auto with_nb(int B, F pick) {
  switch (B) {
    case 0: return pick(std::integral_constant<int, 0>{});
    case 1: return pick(std::integral_constant<int, 1>{});
    case 2: return pick(std::integral_constant<int, 2>{});
    default: return pick(std::integral_constant<int, 3>{});
  }
}

inline size_t ring_bytes(int tensors) { return (size_t)(ring_depth(tensors) + 1) * tensors * kThreads * 16; }

// FinalizeParams of the per-branch host arrays (entries other than parts may be null)
inline int finalize_params(FinalizeParams& p, const float* const* parts, const int* slots, const float* const* gamma,
                           const float* const* beta, float* const* running_mean, float* const* running_var,
                           long long* const* num_batches_tracked, int B) {
  if (B < 1 || B > kMaxBranches) return (int)cudaErrorInvalidValue;
  for (int b = 0; b < B; ++b) {
    if (parts) {
      if (!parts[b] || !slots || slots[b] < 1) return (int)cudaErrorInvalidValue;
      p.parts[b] = parts[b];
      p.slots[b] = slots[b];
    }
    p.gamma[b] = gamma ? gamma[b] : nullptr;
    p.beta[b] = beta ? beta[b] : nullptr;
    p.running_mean[b] = running_mean ? running_mean[b] : nullptr;
    p.running_var[b] = running_var ? running_var[b] : nullptr;
    p.num_batches_tracked[b] = num_batches_tracked ? num_batches_tracked[b] : nullptr;
  }
  p.B = B;
  return 0;
}

// Backward parameters; scratch = [1+B][C] sums followed by the reduction pass' per-block partials (apply reads the sums only)
inline BwdParams bwd_params(const void* dout, const void* u0, const void* u1, const void* u2, int B, const float* scale,
                            const float* shift, const float* mean, const float* rstd, const void* residual, double* scratch,
                            const double* count, void* du0, void* du1, void* du2, void* dres, int M, int C, int act,
                            float slope, int train, int res_after) {
  BwdParams p{};
  p.br = Branches{{(const __nv_bfloat16*)u0, (const __nv_bfloat16*)u1, (const __nv_bfloat16*)u2}, B};
  p.dout = (const __nv_bfloat16*)dout; p.residual = (const __nv_bfloat16*)residual;
  p.scale = scale; p.shift = shift; p.mean = mean; p.rstd = rstd;
  p.sums = scratch; p.part = scratch + (size_t)(1 + B) * C; p.count = count;
  p.du[0] = (__nv_bfloat16*)du0; p.du[1] = (__nv_bfloat16*)du1; p.du[2] = (__nv_bfloat16*)du2;
  p.dres = (__nv_bfloat16*)dres;
  p.M = M; p.C = C; p.act = act; p.slope = slope; p.train = train; p.res_after = res_after;
  return p;
}

// reduction pass + bn_bwd_finalize_kernel: p.sums = (sum dz, sum dz*u_b) over these M rows, parameter gradients written /
// added from them
inline int launch_bwd_reduce(const BwdParams& p, float* dgamma, float* dbeta, float* const* gamma_grad_acc,
                             float* const* beta_grad_acc, int C_logical, cudaStream_t st) {
  const int B = p.br.n, C = p.C;
  const SlabGeo g = SlabGeo::make(C);
  static const int cap_red_env = env_int("HB_BN_CAP_RED", 0);
  static const bool use_occ = env_int("HB_BN_USE_OCC", 1) != 0, occ_debug = env_int("HB_BN_DEBUG", 0) != 0;
  // one branch (Darknet / ReXNet / UNet blocks): ~70 registers and a 48 KB ring -> three resident blocks per SM
  int cap_red = cap_red_env > 0 ? cap_red_env : (B <= 1 ? 3 : 2);
  if (cap_red > 3) cap_red = 3;   // hb_bn_bwd_scratch_doubles sizes the partials for <= 3 blocks per SM
  const size_t smem = sizeof(SlabConsts) + kThreads * 8 * sizeof(float) + ring_bytes(B + 2);
  const auto [kernel, occ] = with_nb(B, [&](auto nb) { return instance<bn_act_bwd_reduce_kernel<decltype(nb)::value>>(smem); });
  if (!occ) return (int)cudaErrorInvalidValue;
  if (occ_debug) fprintf(stderr, "[hb] bn_act_bwd_reduce_kernel<%d> smem %zu: %d resident blocks/SM (cap %d)\n", B, smem, occ, cap_red);
  const dim3 grid = g.grid(p.M, (use_occ && occ < cap_red) ? occ : cap_red);
  kernel<<<grid, kThreads, smem, st>>>(p, g);
  HB_LAUNCH_CHECK();
  BwdFinalizeParams f{};
  f.part = p.part; f.sums = p.sums; f.mean = p.mean; f.rstd = p.rstd; f.dgamma = dgamma; f.dbeta = dbeta;
  for (int b = 0; b < B; ++b) {
    f.gacc[b] = gamma_grad_acc ? gamma_grad_acc[b] : nullptr;
    f.bacc[b] = beta_grad_acc ? beta_grad_acc[b] : nullptr;
  }
  f.nblocks = (int)grid.x; f.B = B; f.C = C; f.C_logical = C_logical > 0 ? C_logical : C;
  bn_bwd_finalize_kernel<<<(C + kFinCh - 1) / kFinCh, dim3(kFinCh, kFinLanes), 0, st>>>(f);
  HB_LAUNCH_CHECK();
  return 0;
}

// apply pass: input gradients from p.sums (and p.count)
inline int launch_bwd_apply(const BwdParams& p, cudaStream_t st) {
  const int B = p.br.n;
  const SlabGeo g = SlabGeo::make(p.C);
  static const int cap_app_env = env_int("HB_BN_CAP_APPLY", 0);
  static const bool use_occ = env_int("HB_BN_USE_OCC", 1) != 0, occ_debug = env_int("HB_BN_DEBUG", 0) != 0;
  const int cap_app = cap_app_env > 0 ? cap_app_env : (B <= 2 ? 3 : 2);   // further limited by the measured occupancy
  const size_t smem = sizeof(SlabConsts) + ring_bytes(B + 2);
  const auto [kernel, occ] = with_nb(B, [&](auto nb) { return instance<bn_act_bwd_apply_kernel<decltype(nb)::value>>(smem); });
  if (!occ) return (int)cudaErrorInvalidValue;
  if (occ_debug) fprintf(stderr, "[hb] bn_act_bwd_apply_kernel<%d> smem %zu: %d resident blocks/SM (cap %d)\n", B, smem, occ, cap_app);
  const dim3 grid = g.grid(p.M, (use_occ && occ < cap_app) ? occ : cap_app);
  kernel<<<grid, kThreads, smem, st>>>(p, g);
  HB_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" {

// Stand-alone statistics pass over u [M, C] bf16 -> parts float [*slots][C][2] (capacity hb_bn_stat_slots_max()).
int hb_bn_stats_partials_bf16(const void* u, int M, int C, float* parts, int* slots, void* stream) {
  if (C % 8 != 0 || !slots) return (int)cudaErrorInvalidValue;
  const SlabGeo g = SlabGeo::make(C);
  static const int min_rows = env_int("HB_BN_STATS_ROWS", 16);
  const dim3 grid = g.grid(M, 4, min_rows);
  *slots = (int)grid.x;
  bn_stats_partials_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)u, M, C, g, parts);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_bn_stat_slots_max(void) { return HB_NUM_SMS * 8; }

int hb_bn_finalize(const float* const* parts, const int* slots, const float* const* gamma, const float* const* beta,
                   float* const* running_mean, float* const* running_var, long long* const* num_batches_tracked,
                   float* mean, float* rstd, float* scale, float* shift, int B, int C, int C_logical, int M, float eps,
                   float momentum, void* stream) {
  FinalizeParams p{};
  if (!parts) return (int)cudaErrorInvalidValue;
  if (const int rc = finalize_params(p, parts, slots, gamma, beta, running_mean, running_var, num_batches_tracked, B))
    return rc;
  p.mean = mean; p.rstd = rstd; p.scale = scale; p.shift = shift;
  p.C = C; p.M = M; p.C_logical = C_logical; p.eps = eps; p.momentum = momentum;
  bn_finalize_kernel<<<dim3((C + kFinCh - 1) / kFinCh, B), dim3(kFinCh, kFinLanes), 0, (cudaStream_t)stream>>>(p);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_bn_partials_sums(const float* const* parts, const int* slots, int B, int C, int C_logical, int M, double* sums,
                        void* stream) {
  FinalizeParams p{};
  if (!parts || !sums) return (int)cudaErrorInvalidValue;
  if (const int rc = finalize_params(p, parts, slots, nullptr, nullptr, nullptr, nullptr, nullptr, B)) return rc;
  p.C = C; p.C_logical = C_logical; p.M = M; p.sums = sums;
  bn_partials_sums_kernel<<<dim3((C + kFinCh - 1) / kFinCh, B), dim3(kFinCh, kFinLanes), 0, (cudaStream_t)stream>>>(p);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_bn_finalize_sums(const double* sums, const float* const* gamma, const float* const* beta,
                        float* const* running_mean, float* const* running_var, long long* const* num_batches_tracked,
                        float* mean, float* rstd, float* scale, float* shift, int B, int C, int C_logical, float eps,
                        float momentum, void* stream) {
  FinalizeParams p{};
  if (!sums) return (int)cudaErrorInvalidValue;
  if (const int rc = finalize_params(p, nullptr, nullptr, gamma, beta, running_mean, running_var, num_batches_tracked, B))
    return rc;
  p.sums = const_cast<double*>(sums);
  p.mean = mean; p.rstd = rstd; p.scale = scale; p.shift = shift;
  p.C = C; p.C_logical = C_logical; p.eps = eps; p.momentum = momentum;
  bn_finalize_sums_kernel<<<dim3((C + 127) / 128, B), 128, 0, (cudaStream_t)stream>>>(p);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_bn_eval_affine(const float* gamma, const float* beta, const float* running_mean, const float* running_var,
                      float eps, int C, int C_logical, float* scale, float* shift, float* mean, float* rstd,
                      void* stream) {
  bn_eval_affine_kernel<<<(C + 127) / 128, 128, 0, (cudaStream_t)stream>>>(gamma, beta, running_mean, running_var, eps,
                                                                            C, C_logical, scale, shift, mean, rstd);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_bn_act_fwd_bf16(const void* u0, const void* u1, const void* u2, int B, const float* scale, const float* shift,
                       const void* residual, void* out, int M, int C, int act, float slope, int res_after,
                       float* out_stats, int* out_stat_slots, void* stream) {
  if (C % 8 != 0 || B < 0 || B > kMaxBranches) return (int)cudaErrorInvalidValue;
  FwdParams p{};
  p.br = Branches{{(const __nv_bfloat16*)u0, (const __nv_bfloat16*)u1, (const __nv_bfloat16*)u2}, B};
  p.scale = scale; p.shift = shift; p.residual = (const __nv_bfloat16*)residual; p.out = (__nv_bfloat16*)out;
  p.M = M; p.C = C; p.act = act; p.slope = slope; p.res_after = res_after;
  if (out_stats && !out_stat_slots) return (int)cudaErrorInvalidValue;
  p.out_stats = out_stats;
  const SlabGeo g = SlabGeo::make(C);
  static const int per_sm_env = env_int("HB_BN_CAP_FWD", 0);
  static const bool use_occ = env_int("HB_BN_USE_OCC", 1) != 0, occ_debug = env_int("HB_BN_DEBUG", 0) != 0;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = ring_bytes(B + 1);
  const auto [kernel, occ] = with_nb(B, [&](auto nb) {
    constexpr int NB = decltype(nb)::value;
    return out_stats ? instance<bn_act_fwd_kernel<NB, true>>(smem) : instance<bn_act_fwd_kernel<NB, false>>(smem);
  });
  if (!occ) return (int)cudaErrorInvalidValue;
  if (occ_debug)
    fprintf(stderr, "[hb] bn_act_fwd_kernel<%d,%d> smem %zu: %d resident blocks/SM\n", B, (int)(out_stats != nullptr), smem, occ);
  // grid = min(4, resident blocks of this instantiation) per SM: registers (launch bound 3) and the ring (48 - 64 KB) decide
  const int fixed = (B + (residual != nullptr) >= 3) ? 3 : 4;
  // <= 4 blocks per SM: the caller's out_stats buffer has 4 x SMs slots (bn_stat_slots)
  const int per_sm = per_sm_env > 0 ? (per_sm_env < 4 ? per_sm_env : 4) : (use_occ ? (occ < 4 ? occ : 4) : fixed);
  const dim3 grid = g.grid(M, per_sm);
  if (out_stat_slots) *out_stat_slots = (int)grid.x;
  kernel<<<grid, kThreads, smem, st>>>(p, g);
  HB_LAUNCH_CHECK();
  return 0;
}

// Backward. scratch: double [hb_bn_bwd_scratch_doubles(M, C, B)], no initialisation needed: [1+B][C] final sums followed
// by the per-block partials of the reduction pass. du_b / dres may be NULL when not needed.
// dgamma/dbeta: fp32 [B][C] outputs (optional); gamma_grad_acc / beta_grad_acc: optional HOST arrays of B device pointers
// (entries may be NULL) to fp32 [C_logical] gradient buffers that dgamma_b / dbeta_b are ADDED to.
size_t hb_bn_bwd_scratch_doubles(int M, int C, int B) {
  const SlabGeo g = SlabGeo::make(C);
  const dim3 grid = g.grid(M, 3);   // upper bound of the reduction pass' row blocks (cap <= 3 per SM)
  return (size_t)(1 + B) * C * (1 + (size_t)grid.x);
}

int hb_bn_act_bwd_bf16(const void* dout, const void* u0, const void* u1, const void* u2, int B, const float* scale,
                       const float* shift, const float* mean, const float* rstd, const void* residual, double* scratch,
                       void* du0, void* du1, void* du2, void* dres, float* dgamma, float* dbeta,
                       float* const* gamma_grad_acc, float* const* beta_grad_acc, int C_logical, int M, int C, int act,
                       float slope, int train, int res_after, void* stream) {
  if (C % 8 != 0 || B < 0 || B > kMaxBranches) return (int)cudaErrorInvalidValue;
  const BwdParams p = bwd_params(dout, u0, u1, u2, B, scale, shift, mean, rstd, residual, scratch, nullptr, du0, du1, du2,
                                 dres, M, C, act, slope, train, res_after);
  const bool want_params = (dgamma && dbeta) || gamma_grad_acc || beta_grad_acc;
  if (train || want_params) {
    const int rc = launch_bwd_reduce(p, dgamma, dbeta, gamma_grad_acc, beta_grad_acc, C_logical, (cudaStream_t)stream);
    if (rc) return rc;
  }
  return launch_bwd_apply(p, (cudaStream_t)stream);
}

int hb_bn_act_bwd_reduce_bf16(const void* dout, const void* u0, const void* u1, const void* u2, int B, const float* scale,
                              const float* shift, const float* mean, const float* rstd, const void* residual,
                              double* scratch, float* dgamma, float* dbeta, float* const* gamma_grad_acc,
                              float* const* beta_grad_acc, int C_logical, int M, int C, int act, float slope, int res_after,
                              void* stream) {
  if (C % 8 != 0 || B < 0 || B > kMaxBranches || !scratch) return (int)cudaErrorInvalidValue;
  const BwdParams p = bwd_params(dout, u0, u1, u2, B, scale, shift, mean, rstd, residual, scratch, nullptr, nullptr, nullptr,
                                 nullptr, nullptr, M, C, act, slope, 1, res_after);
  return launch_bwd_reduce(p, dgamma, dbeta, gamma_grad_acc, beta_grad_acc, C_logical, (cudaStream_t)stream);
}

int hb_bn_act_bwd_apply_bf16(const void* dout, const void* u0, const void* u1, const void* u2, int B, const float* scale,
                             const float* shift, const float* mean, const float* rstd, const void* residual,
                             const double* sums, const double* count, void* du0, void* du1, void* du2, void* dres, int M,
                             int C, int act, float slope, int res_after, void* stream) {
  if (C % 8 != 0 || B < 0 || B > kMaxBranches || !sums || !count) return (int)cudaErrorInvalidValue;
  const BwdParams p = bwd_params(dout, u0, u1, u2, B, scale, shift, mean, rstd, residual, const_cast<double*>(sums), count,
                                 du0, du1, du2, dres, M, C, act, slope, 1, res_after);
  return launch_bwd_apply(p, (cudaStream_t)stream);
}

}  // extern "C"
