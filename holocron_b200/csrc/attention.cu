// SAM and TripletAttention (reference holocron/nn/modules/attention.py:17-30 SAM, :33-56 DimAttention, :59-77
// TripletAttention) over NHWC tensors of bf16 or fp32 storage. The row pitch Cp is a multiple of one 16-byte vector and
// the logical channel count C is passed separately: padding channels never feed a result, and channels C..Cp-1 of every
// output and input gradient are written as zeros. Gates, pooled planes, statistics and parameter gradients are fp32.
//
// SAM: y = x * g, g = sigmoid(w . x + b) per pixel. Forward is one pass (a lane group per pixel row, fixed butterfly
// sum); backward is one pass over x and dy that also writes per-CTA partials of dw and db, added in a fixed order.
//
// TripletAttention: three DimAttention branches that gate x by sigmoid(BN(conv7x7(z_pool(x)))), z_pool taken over C
// (plane H x W), over H (plane C x W) or over W (plane H x C), y = (x g_c + x g_h + x g_w) / 3. The transposes of the
// reference are index arithmetic here:
//   1. pool: one read of x gives all three (max, index, mean) planes. A CTA owns HB rows of one image and walks their
//      W columns: the C reduction is a lane butterfly per pixel, the W reduction runs in shared memory per (h, c), the H
//      reduction is finished per column inside the CTA and written as per-row-block partials that a small kernel
//      combines in block order.
//   2. conv: the 7x7 2->1 zero-padded convolution of each plane on CUDA cores, with per-CTA (sum z, sum z^2) partials
//      for hb_bn_finalize; gate: g = sigmoid(z * scale + shift).
//   3. apply: one read of x and one write of y.
// The backward pass mirrors it: the same pool traversal over x and dy gives sum(dy * x) per plane element, small kernels
// run the sigmoid, BatchNorm and convolution backward (fixed-order partials for dgamma, dbeta and dW, the plane
// gradients in gather form), and one pass writes dx. Max indices follow torch's max(dim).indices (nhwc.cuh). Nothing
// uses atomics or synchronises with the host: every run gives the same bits and the sequence is graph-capturable.
#include "nhwc.cuh"

namespace {

using namespace hb;
using bf16 = __nv_bfloat16;

constexpr int kThreads = 256;
constexpr int kMaxLaneVecs = 4;     // SAM backward: channel vectors per lane (C <= 32 * 4 * V)
constexpr int kSamMaxBlocks = 1024; // SAM backward: partial rows (independent of the device: same bits everywhere)
constexpr int kSlab = 2048;         // triplet pool: HB * Cp bound of the shared per-row state
constexpr int kTaps = 2 * 7 * 7;
constexpr int kBranches = 3;

__device__ __forceinline__ float sigmoid_f(float s) { return 1.f / (1.f + expf(-s)); }

// ------------------------------------------------------------------------------------------------ SAM
// A group of gl lanes per pixel row; lane l holds vectors l, l + gl, ...
template <typename T>
__global__ void __launch_bounds__(kThreads) sam_fwd_kernel(const T* __restrict__ x, const float* __restrict__ w,
                                                           const float* __restrict__ b, T* __restrict__ y,
                                                           float* __restrict__ gate, int R, int C, int Cp, int gl) {
  constexpr int V = Vec16<T>::N;
  const int lane = threadIdx.x % gl;
  const long long r = (long long)blockIdx.x * (kThreads / gl) + threadIdx.x / gl;
  const bool live = r < R;
  const T* xr = x + (size_t)(live ? r : 0) * Cp;
  float s = 0.f;
  if (live) {
    for (int v = lane; v * V < C; v += gl) {
      const Vec16<T> xv = ld16(xr + v * V);
#pragma unroll
      for (int l = 0; l < V; ++l)
        if (v * V + l < C) s = fmaf(w[v * V + l], to_f(xv.v[l]), s);
    }
  }
  s = group_sum(s, gl);
  if (!live) return;
  const float g = sigmoid_f(s + b[0]);
  if (lane == 0) gate[r] = g;
  T* yr = y + (size_t)r * Cp;
  for (int v = lane; v < Cp / V; v += gl) {
    const Vec16<T> xv = ld16(xr + v * V);
    float o[V];
#pragma unroll
    for (int l = 0; l < V; ++l) o[l] = to_f(xv.v[l]) * g;
    st16(yr + v * V, pack<T>(o, v * V, C));
  }
}

// dg = sum_c dy x, ds = dg g (1 - g), dx = dy g + ds w; every group accumulates ds x and ds in registers, the CTA adds
// its groups in order into part[blockIdx.x][0..Cp) (dw) and part[blockIdx.x][Cp] (db).
template <typename T>
__global__ void __launch_bounds__(kThreads) sam_bwd_kernel(const T* __restrict__ x, const T* __restrict__ dy,
                                                           const float* __restrict__ w, const float* __restrict__ gate,
                                                           T* __restrict__ dx, float* __restrict__ part, int R, int C,
                                                           int Cp, int gl) {
  constexpr int V = Vec16<T>::N;
  __shared__ float s_dw[8 * 32 * kMaxLaneVecs * V];   // groups * Cp <= max(256 V, 8 * 32 * kMaxLaneVecs * V)
  __shared__ float s_db[kThreads];
  const int lane = threadIdx.x % gl, grp = threadIdx.x / gl, groups = kThreads / gl;
  const int cv = Cp / V;
  float acc[kMaxLaneVecs][V];
  float dbacc = 0.f;
#pragma unroll
  for (int k = 0; k < kMaxLaneVecs; ++k)
#pragma unroll
    for (int l = 0; l < V; ++l) acc[k][l] = 0.f;
  for (long long base = (long long)blockIdx.x * groups; base < R; base += (long long)gridDim.x * groups) {
    const long long r = base + grp;
    const bool live = r < R;
    Vec16<T> xv[kMaxLaneVecs], gv[kMaxLaneVecs];
    float dg = 0.f;
#pragma unroll
    for (int k = 0; k < kMaxLaneVecs; ++k) {
      const int v = lane + k * gl;
      if (live && v < cv) {
        xv[k] = ld16(x + (size_t)r * Cp + v * V);
        gv[k] = ld16(dy + (size_t)r * Cp + v * V);
#pragma unroll
        for (int l = 0; l < V; ++l)
          if (v * V + l < C) dg = fmaf(to_f(gv[k].v[l]), to_f(xv[k].v[l]), dg);
      }
    }
    dg = group_sum(dg, gl);
    if (!live) continue;
    const float g = gate[r];
    const float ds = dg * (g * (1.f - g));
    dbacc += ds;
#pragma unroll
    for (int k = 0; k < kMaxLaneVecs; ++k) {
      const int v = lane + k * gl;
      if (v >= cv) continue;
      float o[V];
#pragma unroll
      for (int l = 0; l < V; ++l) {
        const int c = v * V + l;
        const float xf = to_f(xv[k].v[l]), gf = to_f(gv[k].v[l]);
        o[l] = c < C ? fmaf(ds, w[c], gf * g) : 0.f;
        if (c < C) acc[k][l] = fmaf(ds, xf, acc[k][l]);
      }
      st16(dx + (size_t)r * Cp + v * V, pack<T>(o, v * V, C));
    }
  }
#pragma unroll
  for (int k = 0; k < kMaxLaneVecs; ++k) {
    const int v = lane + k * gl;
    if (v < cv)
#pragma unroll
      for (int l = 0; l < V; ++l) s_dw[grp * Cp + v * V + l] = acc[k][l];
  }
  if (lane == 0) s_db[grp] = dbacc;
  __syncthreads();
  for (int c = threadIdx.x; c <= Cp; c += kThreads) {
    float t = 0.f;
    for (int q = 0; q < groups; ++q) t += c < Cp ? s_dw[q * Cp + c] : s_db[q];
    part[(size_t)blockIdx.x * (Cp + 1) + c] = t;
  }
}

// column c of part [rows][cols] summed in row order (fp64)
__device__ __forceinline__ float ordered_column_sum(const float* __restrict__ part, int rows, int cols, int c) {
  double t = 0.0;
  for (int r = 0; r < rows; ++r) t += (double)part[(size_t)r * cols + c];
  return (float)t;
}

// out[c] = sum over rows of part[row][c]
__global__ void __launch_bounds__(kThreads) column_sum_kernel(const float* __restrict__ part, int rows, int cols,
                                                              int out_cols, float* __restrict__ out) {
  const int c = blockIdx.x * kThreads + threadIdx.x;
  if (c >= out_cols) return;
  out[c] = ordered_column_sum(part, rows, cols, c);
}

int sam_groups(int dtype, int Cp) { return lane_group(Cp / vec_width(dtype)); }

int sam_blocks(long long R, int gl) {
  const long long need = (R + kThreads / gl - 1) / (kThreads / gl);
  return (int)(need < kSamMaxBlocks ? need : kSamMaxBlocks);
}

bool bad_sam(long long R, int C, int Cp, int dtype) {
  return bad_rows(C, Cp, dtype) || R <= 0 || Cp / vec_width(dtype) > 32 * kMaxLaneVecs;
}

// ------------------------------------------------------------------------------------------------ triplet: pool
struct PoolParams {
  int N, H, W, C, Cp, HB, nHB, gl;
  // forward: pc [N][2][H][W] (max, mean over C) + ic; pw [N][2][H][C] (over W) + iw; hp_* [N][nHB][W][C] partials over
  // the rows of each block (max, sum, index). Backward: pc [N][H][W], pw [N][H][C], hp_sum: sums of dy * x. A null
  // plane pointer disables that branch.
  float* pc; int* ic;
  float* pw; int* iw;
  float* hp_max; float* hp_sum; int* hp_idx;
};

template <typename T, bool kBwd>
__global__ void __launch_bounds__(kThreads) tri_pool_kernel(const T* __restrict__ x, const T* __restrict__ dy,
                                                            PoolParams p) {
  constexpr int V = Vec16<T>::N;
  __shared__ float s_val[kSlab];    // this column's values (backward: dy * x), [row in block][c]
  __shared__ float s_wmax[kSlab];   // running W reduction per (row in block, c)
  __shared__ float s_wsum[kSlab];
  __shared__ int s_widx[kSlab];
  const int n = blockIdx.y, hb = blockIdx.x;
  const int lane = threadIdx.x % p.gl, hl = threadIdx.x / p.gl;
  const int h0 = hb * p.HB, rows = min(p.HB, p.H - h0);
  const int h = h0 + hl;
  const bool live = hl < rows;
  const int cv = p.Cp / V;
  const bool want_c = p.pc != nullptr, want_w = p.pw != nullptr, want_h = p.hp_sum != nullptr;
  if (live)
    for (int v = lane; v < cv; v += p.gl)
#pragma unroll
      for (int l = 0; l < V; ++l) {
        const int o = hl * p.Cp + v * V + l;
        s_wmax[o] = -INFINITY;
        s_wsum[o] = 0.f;
        s_widx[o] = kNoIndex;
      }
  const size_t row_off = (((size_t)n * p.H + (live ? h : 0)) * p.W) * p.Cp;
  for (int w = 0; w < p.W; ++w) {
    float cmax = -INFINITY, csum = 0.f;
    int cidx = kNoIndex;
    if (live) {
      for (int v = lane; v * V < p.C; v += p.gl) {
        const size_t off = row_off + (size_t)w * p.Cp + v * V;
        const Vec16<T> xv = ld16(x + off);
        Vec16<T> gv;
        if (kBwd) gv = ld16(dy + off);
#pragma unroll
        for (int l = 0; l < V; ++l) {
          const int c = v * V + l;
          if (c >= p.C) break;
          const float f = kBwd ? to_f(gv.v[l]) * to_f(xv.v[l]) : to_f(xv.v[l]);
          const int o = hl * p.Cp + c;
          s_val[o] = f;
          if (!kBwd && better(f, c, cmax, cidx)) {
            cmax = f;
            cidx = c;
          }
          csum += f;
          if (want_w) {
            if (!kBwd && better(f, w, s_wmax[o], s_widx[o])) {
              s_wmax[o] = f;
              s_widx[o] = w;
            }
            s_wsum[o] += f;
          }
        }
      }
    }
    // C reduction of pixel (h, w) over the gl lanes of the row
    if (kBwd) csum = group_sum(csum, p.gl);
    else group_max_sum(cmax, cidx, csum, p.gl);
    if (want_c && live && lane == 0) {
      const size_t pix = ((size_t)n * p.H + h) * p.W + w;
      if (kBwd) {
        p.pc[pix] = csum;
      } else {
        const size_t hw = (size_t)p.H * p.W;
        p.pc[(size_t)n * 2 * hw + (size_t)h * p.W + w] = cmax;
        p.pc[(size_t)n * 2 * hw + hw + (size_t)h * p.W + w] = csum / (float)p.C;
        p.ic[pix] = cidx;
      }
    }
    if (want_h) {
      __syncthreads();
      for (int c = threadIdx.x; c < p.C; c += blockDim.x) {
        float m = -INFINITY, s = 0.f;
        int mi = kNoIndex;
        for (int r = 0; r < rows; ++r) {
          const float f = s_val[r * p.Cp + c];
          if (!kBwd && better(f, h0 + r, m, mi)) {
            m = f;
            mi = h0 + r;
          }
          s += f;
        }
        const size_t o = (((size_t)n * p.nHB + hb) * p.W + w) * p.C + c;
        p.hp_sum[o] = s;
        if (!kBwd) {
          p.hp_max[o] = m;
          p.hp_idx[o] = mi;
        }
      }
      __syncthreads();
    }
  }
  if (!want_w || !live) return;
  for (int v = lane; v * V < p.C; v += p.gl)
#pragma unroll
    for (int l = 0; l < V; ++l) {
      const int c = v * V + l;
      if (c >= p.C) break;
      const int o = hl * p.Cp + c;
      const size_t q = ((size_t)n * p.H + h) * p.C + c;
      if (kBwd) {
        p.pw[q] = s_wsum[o];
      } else {
        const size_t hc = (size_t)p.H * p.C;
        p.pw[(size_t)n * 2 * hc + (size_t)h * p.C + c] = s_wmax[o];
        p.pw[(size_t)n * 2 * hc + hc + (size_t)h * p.C + c] = s_wsum[o] / (float)p.W;
        p.iw[q] = s_widx[o];
      }
    }
}

// The H plane from the row-block partials, in block order: forward ph [N][2][C][W] (max, mean) + ih [N][C][W],
// backward ph [N][C][W] (sums). One thread per (n, w, c), c fastest (the partials' order).
template <bool kBwd>
__global__ void __launch_bounds__(kThreads) tri_hcombine_kernel(const float* __restrict__ hp_max,
                                                                const float* __restrict__ hp_sum,
                                                                const int* __restrict__ hp_idx, float* __restrict__ ph,
                                                                int* __restrict__ ih, int N, int H, int W, int C,
                                                                int nHB) {
  const long long e = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (e >= (long long)N * W * C) return;
  const int c = (int)(e % C);
  const int w = (int)((e / C) % W);
  const int n = (int)(e / ((long long)C * W));
  float m = -INFINITY, s = 0.f;
  int mi = kNoIndex;
  for (int b = 0; b < nHB; ++b) {
    const size_t o = (((size_t)n * nHB + b) * W + w) * C + c;
    if (!kBwd && better(hp_max[o], hp_idx[o], m, mi)) {
      m = hp_max[o];
      mi = hp_idx[o];
    }
    s += hp_sum[o];
  }
  const size_t cw = (size_t)C * W;
  if (kBwd) {
    ph[(size_t)n * cw + (size_t)c * W + w] = s;
  } else {
    ph[(size_t)n * 2 * cw + (size_t)c * W + w] = m;
    ph[(size_t)n * 2 * cw + cw + (size_t)c * W + w] = s / (float)H;
    ih[(size_t)n * cw + (size_t)c * W + w] = mi;
  }
}

// ------------------------------------------------------------------------------------------------ triplet: planes
// One launch covers the enabled branches; CTA b belongs to the branch whose block range holds it.
struct Plane {
  const float* in;    // conv: plane [N][2][R][S]; gate: z; bn backward: dG (sums of dy * x)
  const float* aux;   // conv backward: dz; bn backward: z
  const float* aux2;  // bn backward: the gate g
  const float* wt;    // [2][7][7] fp32
  const float* stats; // [mean, rstd, scale, shift]
  float* out;         // conv: z; gate: g; bn backward: dz; conv backward: dplane [N][2][R][S]
  float* part;        // per-CTA partials
  int R, S, first, blocks;
};
struct Planes {
  Plane b[kBranches];
  int N, nb;
  float inv_nb;  // 1 / (number of branches of the layer): the gradient of the final average
  int train;
};

// per-branch output pointers, in the order of the enabled branches
struct PtrArr {
  float* p[kBranches];
};

__device__ __forceinline__ int branch_of(const Planes& q, int blk) {
  int b = 0;
  while (b + 1 < q.nb && blk >= q.b[b + 1].first) ++b;
  return b;
}

__device__ __forceinline__ float* ptr_of(const PtrArr& a, int b) { return b == 0 ? a.p[0] : (b == 1 ? a.p[1] : a.p[2]); }

// q.b[b] through selects: a dynamic index into the launch parameters would copy them to local memory
__device__ __forceinline__ Plane plane_of(const Planes& q, int b) { return b == 0 ? q.b[0] : (b == 1 ? q.b[1] : q.b[2]); }

// z[n, r, s] = sum_{k,i,j} W[k][i][j] P[n, k, r + i - 3, s + j - 3] (zero padding); part[blk] = (sum z, sum z^2)
__global__ void __launch_bounds__(kThreads) tri_conv_fwd_kernel(Planes q) {
  __shared__ float scratch[32];
  __shared__ float s_w[kTaps];
  const int bi = branch_of(q, blockIdx.x);
  const Plane pl = plane_of(q, bi);
  const int blk = blockIdx.x - pl.first;
  for (int t = threadIdx.x; t < kTaps; t += kThreads) s_w[t] = pl.wt[t];
  __syncthreads();
  const long long M = (long long)q.N * pl.R * pl.S;
  const long long e = (long long)blk * kThreads + threadIdx.x;
  float z = 0.f;
  if (e < M) {
    const int s = (int)(e % pl.S), r = (int)((e / pl.S) % pl.R);
    const long long n = e / ((long long)pl.R * pl.S);
    for (int k = 0; k < 2; ++k) {
      const float* P = pl.in + ((size_t)n * 2 + k) * pl.R * pl.S;
#pragma unroll
      for (int i = 0; i < 7; ++i) {
        const int rr = r + i - 3;
        if (rr < 0 || rr >= pl.R) continue;
#pragma unroll
        for (int j = 0; j < 7; ++j) {
          const int ss = s + j - 3;
          if (ss < 0 || ss >= pl.S) continue;
          z = fmaf(s_w[k * 49 + i * 7 + j], P[(size_t)rr * pl.S + ss], z);
        }
      }
    }
    pl.out[e] = z;
  }
  const float sz = block_sum(z, scratch);
  const float sq = block_sum(z * z, scratch);
  if (threadIdx.x == 0) {
    pl.part[(size_t)blk * 2] = sz;
    pl.part[(size_t)blk * 2 + 1] = sq;
  }
}

// g = sigmoid(z * scale + shift)
__global__ void __launch_bounds__(kThreads) tri_gate_kernel(Planes q) {
  const int bi = branch_of(q, blockIdx.x);
  const Plane pl = plane_of(q, bi);
  const long long e = (long long)(blockIdx.x - pl.first) * kThreads + threadIdx.x;
  if (e >= (long long)q.N * pl.R * pl.S) return;
  pl.out[e] = sigmoid_f(fmaf(pl.in[e], pl.stats[2], pl.stats[3]));
}

// dz = (dG / nb) g (1 - g) -> out; part[blk] = (sum dz, sum dz * xhat), xhat = (z - mean) rstd
__global__ void __launch_bounds__(kThreads) tri_bn_bwd_partials_kernel(Planes q) {
  __shared__ float scratch[32];
  const int bi = branch_of(q, blockIdx.x);
  const Plane pl = plane_of(q, bi);
  const int blk = blockIdx.x - pl.first;
  const long long e = (long long)blk * kThreads + threadIdx.x;
  float dz = 0.f, xh = 0.f;
  if (e < (long long)q.N * pl.R * pl.S) {
    const float g = pl.aux2[e];
    dz = pl.in[e] * q.inv_nb * (g * (1.f - g));
    xh = (pl.aux[e] - pl.stats[0]) * pl.stats[1];
    pl.out[e] = dz;
  }
  const float s0 = block_sum(dz, scratch);
  const float s1 = block_sum(dz * xh, scratch);
  if (threadIdx.x == 0) {
    pl.part[(size_t)blk * 2] = s0;
    pl.part[(size_t)blk * 2 + 1] = s1;
  }
}

// dbeta = sum dz, dgamma = sum dz * xhat (one CTA per branch, fixed order) into red[b] = (dgamma, dbeta)
__global__ void __launch_bounds__(kThreads) tri_bn_bwd_reduce_kernel(Planes q, PtrArr dgamma, PtrArr dbeta) {
  __shared__ double scratch[32];
  const Plane pl = plane_of(q, blockIdx.x);
  double s0 = 0.0, s1 = 0.0;
  for (int k = threadIdx.x; k < pl.blocks; k += kThreads) {
    s0 += (double)pl.part[(size_t)k * 2];
    s1 += (double)pl.part[(size_t)k * 2 + 1];
  }
  s0 = block_sum(s0, scratch);
  s1 = block_sum(s1, scratch);
  if (threadIdx.x == 0) {
    ptr_of(dbeta, blockIdx.x)[0] = (float)s0;
    ptr_of(dgamma, blockIdx.x)[0] = (float)s1;
  }
}

// dz of the convolution output: training scale (dz - mean(dz) - xhat mean(dz xhat)), eval scale dz (scale = gamma rstd)
__global__ void __launch_bounds__(kThreads) tri_bn_bwd_apply_kernel(Planes q, PtrArr dgamma,
                                                                    PtrArr dbeta) {
  const int bi = branch_of(q, blockIdx.x);
  const Plane pl = plane_of(q, bi);
  const long long M = (long long)q.N * pl.R * pl.S;
  const long long e = (long long)(blockIdx.x - pl.first) * kThreads + threadIdx.x;
  if (e >= M) return;
  const float dz = pl.out[e];
  float v = dz;
  if (q.train) {
    const float xh = (pl.aux[e] - pl.stats[0]) * pl.stats[1];
    v = dz - ptr_of(dbeta, bi)[0] / (float)M - xh * (ptr_of(dgamma, bi)[0] / (float)M);
  }
  pl.out[e] = v * pl.stats[2];
}

// dP[n, k, r, s] = sum_{i,j} W[k][i][j] dz[n, r - i + 3, s - j + 3] (gather form); part[blk][tap] = the CTA's sum of
// dz[n, r, s] P[n, k, r + i - 3, s + j - 3], a warp butterfly per tap then the warps in order.
__global__ void __launch_bounds__(kThreads) tri_conv_bwd_kernel(Planes q) {
  __shared__ float s_w[kTaps];
  __shared__ float s_red[kThreads / 32][kTaps];
  const int bi = branch_of(q, blockIdx.x);
  const Plane pl = plane_of(q, bi);
  const int blk = blockIdx.x - pl.first;
  for (int t = threadIdx.x; t < kTaps; t += kThreads) s_w[t] = pl.wt[t];
  __syncthreads();
  const long long M = (long long)q.N * pl.R * pl.S;
  const long long e = (long long)blk * kThreads + threadIdx.x;
  const bool live = e < M;
  int r = 0, s = 0;
  long long n = 0;
  float dz = 0.f;
  if (live) {
    s = (int)(e % pl.S);
    r = (int)((e / pl.S) % pl.R);
    n = e / ((long long)pl.R * pl.S);
    dz = pl.aux[e];
  }
  const float* dzn = pl.aux + (size_t)n * pl.R * pl.S;
  for (int k = 0; k < 2; ++k) {
    const float* P = pl.in + ((size_t)n * 2 + k) * pl.R * pl.S;
    float dp = 0.f;
    for (int i = 0; i < 7; ++i) {
      const int rd = r - i + 3, rp = r + i - 3;
      for (int j = 0; j < 7; ++j) {
        const int sd = s - j + 3, sp = s + j - 3;
        if (live && rd >= 0 && rd < pl.R && sd >= 0 && sd < pl.S)
          dp = fmaf(s_w[k * 49 + i * 7 + j], dzn[(size_t)rd * pl.S + sd], dp);
        float t = (live && rp >= 0 && rp < pl.R && sp >= 0 && sp < pl.S) ? dz * P[(size_t)rp * pl.S + sp] : 0.f;
        t = warp_sum(t);
        if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5][k * 49 + i * 7 + j] = t;
      }
    }
    if (live) pl.out[((size_t)n * 2 + k) * pl.R * pl.S + (size_t)r * pl.S + s] = dp;
  }
  __syncthreads();
  for (int t = threadIdx.x; t < kTaps; t += kThreads) {
    float a = 0.f;
    for (int wv = 0; wv < kThreads / 32; ++wv) a += s_red[wv][t];
    pl.part[(size_t)blk * kTaps + t] = a;
  }
}

// dW[b][tap] = sum over the branch's CTAs of part[blk][tap], in order (fp64); one CTA per branch
__global__ void __launch_bounds__(128) tri_wgrad_reduce_kernel(Planes q, PtrArr dw) {
  const Plane pl = plane_of(q, blockIdx.x);
  const int t = threadIdx.x;
  if (t >= kTaps) return;
  ptr_of(dw, blockIdx.x)[t] = ordered_column_sum(pl.part, pl.blocks, kTaps, t);
}

// ------------------------------------------------------------------------------------------------ triplet: x passes
struct XParams {
  const float *gc, *gh, *gw;     // gates [N][H][W], [N][C][W], [N][H][C] (null: branch disabled)
  const float *dpc, *dph, *dpw;  // backward: plane gradients [N][2][..]
  const int *ic, *ih, *iw;       // backward: max indices
  int N, H, W, C, Cp;
  float nb;
};

// y = (x g_c + x g_h + x g_w) / nb over the enabled branches, in that order
template <typename T>
__global__ void __launch_bounds__(kThreads) tri_apply_kernel(const T* __restrict__ x, T* __restrict__ y, XParams p) {
  constexpr int V = Vec16<T>::N;
  const int cv = p.Cp / V;
  const long long total = (long long)p.N * p.H * p.W * cv;
  for (long long e = (long long)blockIdx.x * kThreads + threadIdx.x; e < total; e += (long long)gridDim.x * kThreads) {
    const int c0 = (int)(e % cv) * V;
    const long long pix = e / cv;
    const int w = (int)(pix % p.W), h = (int)((pix / p.W) % p.H);
    const long long n = pix / ((long long)p.W * p.H);
    const Vec16<T> xv = ld16(x + (size_t)e * V);
    const float gc = p.gc ? p.gc[pix] : 0.f;
    float o[V];
#pragma unroll
    for (int l = 0; l < V; ++l) {
      const int c = c0 + l;
      if (c >= p.C) {
        o[l] = 0.f;
        continue;
      }
      const float xf = to_f(xv.v[l]);
      float s = 0.f;
      bool first = true;
      if (p.gc) { s = xf * gc; first = false; }
      if (p.gh) { const float t = xf * p.gh[((size_t)n * p.C + c) * p.W + w]; s = first ? t : s + t; first = false; }
      if (p.gw) { const float t = xf * p.gw[((size_t)n * p.H + h) * p.C + c]; s = first ? t : s + t; }
      o[l] = s / p.nb;
    }
    st16(y + (size_t)e * V, pack<T>(o, c0, p.C));
  }
}

// dx = dy (g_c + g_h + g_w) / nb + for each branch: dmax at the saved index + dmean / L
template <typename T>
__global__ void __launch_bounds__(kThreads) tri_dx_kernel(const T* __restrict__ dy, T* __restrict__ dx, XParams p) {
  constexpr int V = Vec16<T>::N;
  const int cv = p.Cp / V;
  const long long total = (long long)p.N * p.H * p.W * cv;
  const size_t hw = (size_t)p.H * p.W, cw = (size_t)p.C * p.W, hc = (size_t)p.H * p.C;
  for (long long e = (long long)blockIdx.x * kThreads + threadIdx.x; e < total; e += (long long)gridDim.x * kThreads) {
    const int c0 = (int)(e % cv) * V;
    const long long pix = e / cv;
    const int w = (int)(pix % p.W), h = (int)((pix / p.W) % p.H);
    const size_t n = (size_t)(pix / ((long long)p.W * p.H));
    const Vec16<T> gv = ld16(dy + (size_t)e * V);
    float gc = 0.f, cmax = 0.f, cmean = 0.f;
    int cidx = -1;
    if (p.gc) {
      gc = p.gc[pix];
      cidx = p.ic[pix];
      cmax = p.dpc[n * 2 * hw + (size_t)h * p.W + w];
      cmean = p.dpc[n * 2 * hw + hw + (size_t)h * p.W + w] / (float)p.C;
    }
    float o[V];
#pragma unroll
    for (int l = 0; l < V; ++l) {
      const int c = c0 + l;
      if (c >= p.C) {
        o[l] = 0.f;
        continue;
      }
      float g = gc;
      float d = 0.f;
      if (p.gc) d = (cidx == c ? cmax : 0.f) + cmean;
      if (p.gh) {
        const size_t q = n * cw + (size_t)c * p.W + w;
        g += p.gh[q];
        d += (p.ih[q] == h ? p.dph[n * 2 * cw + (size_t)c * p.W + w] : 0.f) +
             p.dph[n * 2 * cw + cw + (size_t)c * p.W + w] / (float)p.H;
      }
      if (p.gw) {
        const size_t q = n * hc + (size_t)h * p.C + c;
        g += p.gw[q];
        d += (p.iw[q] == w ? p.dpw[n * 2 * hc + (size_t)h * p.C + c] : 0.f) +
             p.dpw[n * 2 * hc + hc + (size_t)h * p.C + c] / (float)p.W;
      }
      o[l] = fmaf(to_f(gv.v[l]), g / p.nb, d);
    }
    st16(dx + (size_t)e * V, pack<T>(o, c0, p.C));
  }
}

// rows per CTA of the pool pass: the lane groups of a CTA, bounded by the shared per-row state
int tri_row_block(int H, int Cp, int dtype) {
  int hb = kThreads / lane_group(Cp / vec_width(dtype));
  if (hb * Cp > kSlab) hb = kSlab / Cp;
  return hb < H ? hb : H;
}

bool bad_triplet(int N, int H, int W, int C, int Cp, int dtype) {
  return bad_rows(C, Cp, dtype) || N <= 0 || H <= 0 || W <= 0 || Cp > kSlab || (long long)N * H * W * Cp >= (1LL << 40) ||
         N > 65535;
}

template <typename T>
int launch_pool(bool bwd, const void* x, const void* dy, PoolParams p, float* ph, int* ih, cudaStream_t st) {
  const dim3 grid((unsigned)p.nHB, (unsigned)p.N);
  if (bwd) tri_pool_kernel<T, true><<<grid, kThreads, 0, st>>>((const T*)x, (const T*)dy, p);
  else tri_pool_kernel<T, false><<<grid, kThreads, 0, st>>>((const T*)x, nullptr, p);
  HB_LAUNCH_CHECK();
  if (p.hp_sum) {
    const long long total = (long long)p.N * p.W * p.C;
    const unsigned g = (unsigned)((total + kThreads - 1) / kThreads);
    if (bwd) tri_hcombine_kernel<true><<<g, kThreads, 0, st>>>(nullptr, p.hp_sum, nullptr, ph, nullptr, p.N, p.H, p.W,
                                                               p.C, p.nHB);
    else tri_hcombine_kernel<false><<<g, kThreads, 0, st>>>(p.hp_max, p.hp_sum, p.hp_idx, ph, ih, p.N, p.H, p.W, p.C,
                                                            p.nHB);
    HB_LAUNCH_CHECK();
  }
  return 0;
}

int make_pool(PoolParams& p, int N, int H, int W, int C, int Cp, int dtype) {
  if (bad_triplet(N, H, W, C, Cp, dtype)) return (int)cudaErrorInvalidValue;
  p = PoolParams{};
  p.N = N; p.H = H; p.W = W; p.C = C; p.Cp = Cp;
  p.gl = lane_group(Cp / vec_width(dtype));
  p.HB = tri_row_block(H, Cp, dtype);
  p.nHB = (H + p.HB - 1) / p.HB;
  return 0;
}

// fills q from host arrays of per-branch pointers; a branch without `in` is disabled. 0 or cudaErrorInvalidValue
int make_planes(Planes& q, const float* const* in, const float* const* aux, const float* const* aux2,
                const float* const* wt, const float* const* stats, float* const* out, float* const* part,
                const int* rows, const int* cols, int N) {
  if (!in || !out || !rows || !cols || N <= 0) return (int)cudaErrorInvalidValue;
  q = Planes{};
  q.N = N;
  int first = 0;
  for (int b = 0; b < kBranches; ++b) {
    if (!in[b]) continue;
    if (rows[b] <= 0 || cols[b] <= 0 || !out[b]) return (int)cudaErrorInvalidValue;
    Plane& pl = q.b[q.nb++];
    pl.in = in[b];
    pl.aux = aux ? aux[b] : nullptr;
    pl.aux2 = aux2 ? aux2[b] : nullptr;
    pl.wt = wt ? wt[b] : nullptr;
    pl.stats = stats ? stats[b] : nullptr;
    pl.out = out[b];
    pl.part = part ? part[b] : nullptr;
    pl.R = rows[b];
    pl.S = cols[b];
    const long long M = (long long)N * rows[b] * cols[b];
    pl.first = first;
    pl.blocks = (int)((M + kThreads - 1) / kThreads);
    first += pl.blocks;
  }
  return q.nb ? 0 : (int)cudaErrorInvalidValue;
}

int total_blocks(const Planes& q) { return q.b[q.nb - 1].first + q.b[q.nb - 1].blocks; }

}  // namespace

extern "C" {

int hb_sam_bwd_slots(int R, int C, int Cp, int dtype) {
  if (bad_sam(R, C, Cp, dtype)) return 0;
  return sam_blocks(R, sam_groups(dtype, Cp));
}

int hb_sam_fwd(const void* x, const float* w, const float* b, void* y, float* gate, int R, int C, int Cp, int dtype,
               void* stream) {
  if (bad_sam(R, C, Cp, dtype)) return (int)cudaErrorInvalidValue;
  const int gl = sam_groups(dtype, Cp);
  const unsigned grid = (unsigned)(((long long)R * gl + kThreads - 1) / kThreads);
  return with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    sam_fwd_kernel<T><<<grid, kThreads, 0, (cudaStream_t)stream>>>((const T*)x, w, b, (T*)y, gate, R, C, Cp, gl);
    HB_LAUNCH_CHECK();
    return 0;
  });
}

int hb_sam_bwd(const void* x, const void* dy, const float* w, const float* gate, void* dx, float* part, float* dwdb,
               int R, int C, int Cp, int dtype, void* stream) {
  if (bad_sam(R, C, Cp, dtype)) return (int)cudaErrorInvalidValue;
  const int gl = sam_groups(dtype, Cp);
  const int blocks = sam_blocks(R, gl);
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = with_dtype(dtype, [&](auto t) {
        using T = decltype(t);
        sam_bwd_kernel<T><<<blocks, kThreads, 0, st>>>((const T*)x, (const T*)dy, w, gate, (T*)dx, part, R, C, Cp, gl);
        HB_LAUNCH_CHECK();
        return 0;
      }))
    return rc;
  // dwdb[0..C) = dw, dwdb[C] = db: the dw columns, then the db column moved next to them
  column_sum_kernel<<<(C + kThreads - 1) / kThreads, kThreads, 0, st>>>(part, blocks, Cp + 1, C, dwdb);
  HB_LAUNCH_CHECK();
  column_sum_kernel<<<1, kThreads, 0, st>>>(part + Cp, blocks, Cp + 1, 1, dwdb + C);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_triplet_row_block(int H, int C, int Cp, int dtype) {
  if (bad_triplet(1, H, 1, C, Cp, dtype)) return 0;
  return tri_row_block(H, Cp, dtype);
}

int hb_triplet_pool_fwd(const void* x, float* pc, int* ic, float* pw, int* iw, float* hp_max, float* hp_sum,
                        int* hp_idx, float* ph, int* ih, int N, int H, int W, int C, int Cp, int dtype, void* stream) {
  PoolParams p;
  if (int rc = make_pool(p, N, H, W, C, Cp, dtype)) return rc;
  if ((pc && !ic) || (pw && !iw) || (ph && (!ih || !hp_max || !hp_sum || !hp_idx)) || (!pc && !pw && !ph))
    return (int)cudaErrorInvalidValue;
  p.pc = pc; p.ic = ic; p.pw = pw; p.iw = iw;
  if (ph) { p.hp_max = hp_max; p.hp_sum = hp_sum; p.hp_idx = hp_idx; }
  return with_dtype(dtype, [&](auto t) {
    return launch_pool<decltype(t)>(false, x, nullptr, p, ph, ih, (cudaStream_t)stream);
  });
}

int hb_triplet_pool_bwd(const void* x, const void* dy, float* dgc, float* dgw, float* hp_sum, float* dgh, int N, int H,
                        int W, int C, int Cp, int dtype, void* stream) {
  PoolParams p;
  if (int rc = make_pool(p, N, H, W, C, Cp, dtype)) return rc;
  if ((dgh && !hp_sum) || (!dgc && !dgw && !dgh)) return (int)cudaErrorInvalidValue;
  p.pc = dgc; p.pw = dgw;
  if (dgh) p.hp_sum = hp_sum;
  return with_dtype(dtype, [&](auto t) {
    return launch_pool<decltype(t)>(true, x, dy, p, dgh, nullptr, (cudaStream_t)stream);
  });
}

int hb_triplet_conv_fwd(const float* const* plane, const float* const* weight, float* const* z, float* const* parts,
                        int* slots, const int* rows, const int* cols, int N, void* stream) {
  Planes q;
  if (int rc = make_planes(q, plane, nullptr, nullptr, weight, nullptr, z, parts, rows, cols, N)) return rc;
  for (int b = 0, k = 0; b < kBranches; ++b) {
    if (!plane[b]) continue;
    if (!weight || !weight[b] || !parts || !parts[b]) return (int)cudaErrorInvalidValue;
    if (slots) slots[b] = q.b[k++].blocks;
  }
  tri_conv_fwd_kernel<<<total_blocks(q), kThreads, 0, (cudaStream_t)stream>>>(q);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_triplet_gate(const float* const* z, const float* const* stats, float* const* gate, const int* rows,
                    const int* cols, int N, void* stream) {
  Planes q;
  if (int rc = make_planes(q, z, nullptr, nullptr, nullptr, stats, gate, nullptr, rows, cols, N)) return rc;
  for (int b = 0; b < kBranches; ++b)
    if (z[b] && (!stats || !stats[b])) return (int)cudaErrorInvalidValue;
  tri_gate_kernel<<<total_blocks(q), kThreads, 0, (cudaStream_t)stream>>>(q);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_triplet_bn_bwd(const float* const* dg, const float* const* z, const float* const* gate,
                      const float* const* stats, float* const* dz, float* const* parts, float* const* dgamma,
                      float* const* dbeta, const int* rows, const int* cols, int N, float inv_nb, int train,
                      void* stream) {
  Planes q;
  if (int rc = make_planes(q, dg, z, gate, nullptr, stats, dz, parts, rows, cols, N)) return rc;
  PtrArr dga{}, dba{};
  for (int b = 0, k = 0; b < kBranches; ++b) {
    if (!dg[b]) continue;
    if (!z || !z[b] || !gate || !gate[b] || !stats || !stats[b] || !parts || !parts[b] || !dgamma || !dgamma[b] ||
        !dbeta || !dbeta[b])
      return (int)cudaErrorInvalidValue;
    dga.p[k] = dgamma[b];
    dba.p[k] = dbeta[b];
    ++k;
  }
  q.inv_nb = inv_nb;
  q.train = train;
  cudaStream_t st = (cudaStream_t)stream;
  const int blocks = total_blocks(q);
  tri_bn_bwd_partials_kernel<<<blocks, kThreads, 0, st>>>(q);
  HB_LAUNCH_CHECK();
  tri_bn_bwd_reduce_kernel<<<q.nb, kThreads, 0, st>>>(q, dga, dba);
  HB_LAUNCH_CHECK();
  tri_bn_bwd_apply_kernel<<<blocks, kThreads, 0, st>>>(q, dga, dba);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_triplet_conv_bwd(const float* const* plane, const float* const* weight, const float* const* dz,
                        float* const* dplane, float* const* parts, float* const* dweight, const int* rows,
                        const int* cols, int N, void* stream) {
  Planes q;
  if (int rc = make_planes(q, plane, dz, nullptr, weight, nullptr, dplane, parts, rows, cols, N)) return rc;
  PtrArr dwa{};
  for (int b = 0, k = 0; b < kBranches; ++b) {
    if (!plane[b]) continue;
    if (!weight || !weight[b] || !dz || !dz[b] || !parts || !parts[b] || !dweight || !dweight[b])
      return (int)cudaErrorInvalidValue;
    dwa.p[k++] = dweight[b];
  }
  cudaStream_t st = (cudaStream_t)stream;
  tri_conv_bwd_kernel<<<total_blocks(q), kThreads, 0, st>>>(q);
  HB_LAUNCH_CHECK();
  tri_wgrad_reduce_kernel<<<q.nb, 128, 0, st>>>(q, dwa);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_triplet_apply(const void* x, void* y, const float* gc, const float* gh, const float* gw, int N, int H, int W,
                     int C, int Cp, int dtype, void* stream) {
  if (bad_triplet(N, H, W, C, Cp, dtype) || (!gc && !gh && !gw)) return (int)cudaErrorInvalidValue;
  XParams p{};
  p.gc = gc; p.gh = gh; p.gw = gw;
  p.N = N; p.H = H; p.W = W; p.C = C; p.Cp = Cp;
  p.nb = (float)((gc != nullptr) + (gh != nullptr) + (gw != nullptr));
  const size_t total = (size_t)N * H * W * (Cp / vec_width(dtype));
  const int grid = stream_grid(total, kThreads, 16);
  return with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    tri_apply_kernel<T><<<grid, kThreads, 0, (cudaStream_t)stream>>>((const T*)x, (T*)y, p);
    HB_LAUNCH_CHECK();
    return 0;
  });
}

int hb_triplet_dx(const void* dy, void* dx, const float* gc, const float* gh, const float* gw, const float* dpc,
                  const float* dph, const float* dpw, const int* ic, const int* ih, const int* iw, int N, int H, int W,
                  int C, int Cp, int dtype, void* stream) {
  if (bad_triplet(N, H, W, C, Cp, dtype) || (!gc && !gh && !gw) || (gc && (!dpc || !ic)) || (gh && (!dph || !ih)) ||
      (gw && (!dpw || !iw)))
    return (int)cudaErrorInvalidValue;
  XParams p{};
  p.gc = gc; p.gh = gh; p.gw = gw;
  p.dpc = dpc; p.dph = dph; p.dpw = dpw;
  p.ic = ic; p.ih = ih; p.iw = iw;
  p.N = N; p.H = H; p.W = W; p.C = C; p.Cp = Cp;
  p.nb = (float)((gc != nullptr) + (gh != nullptr) + (gw != nullptr));
  const size_t total = (size_t)N * H * W * (Cp / vec_width(dtype));
  const int grid = stream_grid(total, kThreads, 16);
  return with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    tri_dx_kernel<T><<<grid, kThreads, 0, (cudaStream_t)stream>>>((const T*)dy, (T*)dx, p);
    HB_LAUNCH_CHECK();
    return 0;
  });
}

}  // extern "C"
