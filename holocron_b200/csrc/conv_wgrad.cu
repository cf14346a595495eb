// Weight-gradient of a 2-D convolution on the sm_90a tensor cores (wgmma).
//
//   dW[co, r, s, ci] = sum_m dY[m, co] * X[pix(m) + (r, s), ci]        (m over all N*Ho*Wo output pixels)
//
// GEMM view per filter tap: D[M = co][N = ci] += A[co, m] * B[ci, m] with the reduction (K) dimension being the
// output pixels. Both operands are "MN-major" in shared memory (the pixel index is the slow one), which wgmma
// supports directly for 16-bit types (transposed operands), so dY ([M_total, Cout] row-major) and the im2col view of X
// are loaded by TMA exactly as they sit in HBM - no transposes:
//   A stage = 64 pixels x 128 co   (two 64-wide TMA boxes, 128B-swizzled rows = pixels; one per consumer warpgroup)
//   B stage = 64 pixels x Cin-tile (im2col TMA: padding / stride / row wrap handled in hardware)
// The planner splits the work into (co tile, ci tile, tap, pixel range) units. A CTA runs up to T = 3 units that differ
// only in tap at once: per stage it loads the dY boxes once and one im2col box per tap, and issues one wgmma per tap on
// the same A descriptor, so each dY byte moved into shared memory feeds T taps. Each tap's accumulators (64 co x <= 128
// ci per warpgroup) live in registers and see the same k-steps in the same order as a one-tap unit, so dW does not
// depend on T. Results are reduced across pixel ranges with fp32 red.global.add, written as per-range partials for a
// fixed-order reduction, or stored directly when there is a single range.
// This replaces cuDNN's wgrad behind autograd for nn.Conv2d in the reference
// (holocron/models/utils.py:71, models/classification/repvgg.py:55-62).
#include <cstdlib>
#include "conv_common.cuh"

namespace {

using namespace tc;
using namespace conv;

constexpr int kBKpix = 64;     // pixels (reduction) per stage
constexpr int kChunkBytes = kBKpix * 128;  // one 64px x 64ch box = 8 KiB
constexpr int kABytes = 2 * kChunkBytes;   // 128 co
constexpr int kMaxTaps = 3;                // 3 x 64 accumulators per thread at CIW = 128 (232 registers after setmaxnreg)
constexpr int kProducerRegs = 40;          // per thread after setmaxnreg: 128 x (40 + 2 x 232) = 64 512 <= 64 K registers
constexpr int kConsumerRegs = 232;

struct WgradParams {
  int m_total, Ho, Wo, stride, pad, dil, R, S, Cin, Cout;
  int ci_tile;         // Cin tile (<= 128)
  int ci_chunks;       // ceil(ci_tile / 64)
  int taps_per_group;  // taps a CTA runs together (1 as planned; the launcher regroups them, see group_taps)
  int num_tap_groups, num_co_tiles, num_ci_tiles, k_splits;
  int kblocks_total;   // ceil(m_total / 64)
  int stages, stage_bytes;
  int use_atomics;     // 0: single pixel range, store; 1: atomics; 2: per-range partials in `ws` (reduced by a 2nd kernel)
  float* dw;           // [Cout, R, S, Cin] fp32
  float* ws;           // [k_splits][Cout*R*S*Cin] fp32 partial sums (mode 2)
  long long dw_elems;
};

// CIW: the Cin tile rounded up to 16 (16 ... 128) = the MMA widths of its 64-channel chunks: min(CIW, 64), then CIW - 64.
// T: taps per work item (p.taps_per_group); the last tap group of a filter may hold fewer (RS % T).
template <int CIW, int T>
__global__ void __launch_bounds__(kThreads, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap tmDY, const __grid_constant__ CUtensorMap tmX, const WgradParams p) {
  constexpr int kChunks = (CIW + 63) / 64, kNLast = CIW - 64 * (kChunks - 1);
  constexpr int kBTapBytes = kChunks * kChunkBytes;   // one tap's im2col boxes in a stage
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)p.stages * p.stage_bytes);
  uint64_t* empty_bar = full_bar + p.stages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmDY);
    prefetch_tmap(&tmX);
    for (int i = 0; i < p.stages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kConsumers / 32); }
    fence_barrier_init();
  }
  __syncthreads();

  const int RS = p.R * p.S;
  const int num_units = p.num_co_tiles * p.num_ci_tiles * p.num_tap_groups * p.k_splits;

  // work-item decode (an item is the units of one tap group): k_split fastest so neighbouring CTAs share the same filter
  // slab / write target
  auto decode = [&](int unit, int& co_t, int& ci_t, int& tg, int& ks) {
    ks = unit % p.k_splits; unit /= p.k_splits;
    tg = unit % p.num_tap_groups; unit /= p.num_tap_groups;
    ci_t = unit % p.num_ci_tiles; co_t = unit / p.num_ci_tiles;
  };
  auto kb_range = [&](int ks, int& kb0, int& kb1) {
    const int per = (p.kblocks_total + p.k_splits - 1) / p.k_splits;
    kb0 = ks * per;
    kb1 = min(kb0 + per, p.kblocks_total);
  };

  if (warp < 4) {
    regs_release<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      Ring ring;
      for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
        int co_t, ci_t, tg, ks, kb0, kb1;
        decode(unit, co_t, ci_t, tg, ks);
        kb_range(ks, kb0, kb1);
        const int tap0 = tg * T;
        const int ntaps = min(T, RS - tap0);
        const uint32_t tx = kABytes + ntaps * kBTapBytes;
        for (int kb = kb0; kb < kb1; ++kb) {
          const int m0 = kb * kBKpix;
          const int q0 = m0 % p.Wo, p0 = (m0 / p.Wo) % p.Ho, n0 = m0 / (p.Wo * p.Ho);
          const int base_w = q0 * p.stride - p.pad, base_h = p0 * p.stride - p.pad;
          uint64_t* bar = &full_bar[ring.stage];
          mbar_wait(&empty_bar[ring.stage], ring.phase ^ 1);
          uint8_t* sa = smem + (size_t)ring.stage * p.stage_bytes;
          mbar_arrive_expect_tx(bar, tx);
          tma_load_2d(&tmDY, bar, sa, co_t * 128, m0);
          tma_load_2d(&tmDY, bar, sa + kChunkBytes, co_t * 128 + 64, m0);
          for (int t = 0; t < ntaps; ++t) {
            const int tap = tap0 + t, r = tap / p.S, s = tap % p.S;
            uint8_t* sb = sa + kABytes + t * kBTapBytes;
            for (int c = 0; c < kChunks; ++c)
              tma_load_im2col_4d(&tmX, bar, sb + c * kChunkBytes, ci_t * p.ci_tile + c * 64, base_w, base_h, n0,
                                 (uint16_t)(s * p.dil), (uint16_t)(r * p.dil));
          }
          ring.next(p.stages);
        }
      }
    }
    return;
  }

  // ================= consumers: warpgroup wg owns output channels [64*wg, 64*wg + 64) of the co tile =================
  regs_acquire<kConsumerRegs>();
  const int et = threadIdx.x - 128;
  const int wg = et >> 7;
  const int frow = frag_row(et & 127), fcol = frag_col(et & 127);
  const uint32_t dhi = desc_hi(1024);
  float acc[T][CIW / 2];   // per tap: [chunk 0: 32 | chunk 1: kNLast / 2]
  Ring ring;
  // The pixel range [kb0, kb1) of NT taps: one commit group per stage, every tap's MMAs on the same A descriptor. NT is
  // a template argument so that each fence -> commit region is straight-line (a tap group shorter than T is its own
  // instantiation, picked by a branch outside the region).
  auto mainloop = [&](auto nt, int kb0, int kb1) {
    constexpr int NT = decltype(nt)::value;
    int prev = -1;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full_bar[ring.stage], ring.phase);
      // 16 pixels = two 8-row swizzle atoms (SBO 1024 B), i.e. 2048 B per k-step
      const uint32_t s_lo = desc_lo(smem_u32(smem + (size_t)ring.stage * p.stage_bytes), 16);
      const uint32_t a_lo = s_lo + (uint32_t)wg * (kChunkBytes >> 4);
      const uint32_t b_lo = s_lo + (kABytes >> 4);
      const uint32_t acc0 = kb > kb0 ? 1u : 0u;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBKpix / 16; ++k) {
        const uint64_t ad = make_desc(a_lo + k * (2048 >> 4), dhi);
        const uint32_t sc = acc0 | (uint32_t)k;
#pragma unroll
        for (int t = 0; t < NT; ++t) {
          const uint32_t bt = b_lo + t * (kBTapBytes >> 4) + k * (2048 >> 4);
          if constexpr (kChunks == 1) {
            wgmma<kNLast, 1, 1>(acc[t], ad, make_desc(bt, dhi), sc);
          } else {
            wgmma<64, 1, 1>(acc[t], ad, make_desc(bt, dhi), sc);
            wgmma<kNLast, 1, 1>(acc[t] + 32, ad, make_desc(bt + (kChunkBytes >> 4), dhi), sc);
          }
        }
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = ring.stage;
      ring.next(p.stages);
    }
    wgmma_wait<0>();
#pragma unroll
    for (int t = 0; t < NT; ++t) fence_regs(acc[t]);
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
  };

  for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
    int co_t, ci_t, tg, ks, kb0, kb1;
    decode(unit, co_t, ci_t, tg, ks);
    kb_range(ks, kb0, kb1);
    const int tap0 = tg * T;
    const int ntaps = min(T, RS - tap0);
    if (ntaps == T) {
      mainloop(std::integral_constant<int, T>{}, kb0, kb1);
    } else if constexpr (T == 3) {
      if (ntaps == 2) mainloop(std::integral_constant<int, 2>{}, kb0, kb1);
      else mainloop(std::integral_constant<int, 1>{}, kb0, kb1);
    } else if constexpr (T == 2) {
      mainloop(std::integral_constant<int, 1>{}, kb0, kb1);
    }

    const bool have = kb1 > kb0;   // empty pixel range: this unit's slice of the partial buffer must still read as zero
    if (!have && p.use_atomics != 2) continue;
    float* base = p.use_atomics == 2 ? p.ws + (size_t)ks * p.dw_elems : p.dw;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int co = co_t * 128 + 64 * wg + frow + 8 * h;
      if (co >= p.Cout) continue;
#pragma unroll
      for (int t = 0; t < T; ++t) {
        if (t >= ntaps) break;
        float* drow = base + ((size_t)co * RS + tap0 + t) * p.Cin;
#pragma unroll
        for (int j = 0; j < CIW / 8; ++j) {
          // register block j: chunk j / 8, columns 8 * (j % 8) + fcol of that chunk
          const int c = (j >> 3) * 64 + 8 * (j & 7) + fcol;
          const int ci = ci_t * p.ci_tile + c;
          if (c >= p.ci_tile || ci >= p.Cin) continue;
          const float v0 = have ? acc[t][4 * j + 2 * h] : 0.f, v1 = have ? acc[t][4 * j + 2 * h + 1] : 0.f;
          if (p.use_atomics == 1) {
            atomicAdd(drow + ci, v0);
            atomicAdd(drow + ci + 1, v1);
          } else {
            *reinterpret_cast<float2*>(drow + ci) = make_float2(v0, v1);   // Cin % 8 == 0 and ci even: 8-byte aligned
          }
        }
      }
    }
  }
}

// dw[i] = sum_k ws[k][i] in a fixed order (deterministic). blockDim = (32, 8): threadIdx.x walks float4 columns,
// threadIdx.y takes the slices k = y, y+8, ...; the 8 partial sums are combined through shared memory in y order.
// (A single thread per column walking a hundred or more slices serially is latency-bound, not bandwidth-bound.)
// Elements [0, n_first) go to dw, [n_first, n) to dw2 (two gradient tensors filled by one launch; n_first % 4 == 0);
// accumulate != 0: dw += sum instead of dw = sum (gradient accumulation straight into the parameter's .grad storage, what
// autograd's AccumulateGrad would do with one more element-wise kernel per parameter and step).
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ dw, long long n,
                                                           int k_splits, float* __restrict__ dw2, long long n_first,
                                                           int accumulate) {
  __shared__ float4 part[8][32];
  const long long i4 = ((long long)blockIdx.x * 32 + threadIdx.x) * 4;
  const int y = threadIdx.y;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i4 + 3 < n) {
#pragma unroll 4
    for (int k = y; k < k_splits; k += 8) {
      const float4 v = *reinterpret_cast<const float4*>(ws + (size_t)k * n + i4);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  } else if (i4 < n) {
    float t[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k = y; k < k_splits; k += 8)
      for (int j = 0; j < 4 && i4 + j < n; ++j) t[j] += ws[(size_t)k * n + i4 + j];
    acc = make_float4(t[0], t[1], t[2], t[3]);
  }
  part[y][threadIdx.x] = acc;
  __syncthreads();
  if (y == 0 && i4 < n) {
    float4 r = part[0][threadIdx.x];
#pragma unroll
    for (int j = 1; j < 8; ++j) {
      const float4 v = part[j][threadIdx.x];
      r.x += v.x; r.y += v.y; r.z += v.z; r.w += v.w;
    }
    float* dst = i4 < n_first ? dw + i4 : dw2 + (i4 - n_first);
    if (i4 + 3 < n) {
      if (accumulate) {
        const float4 o = *reinterpret_cast<const float4*>(dst);
        r.x += o.x; r.y += o.y; r.z += o.z; r.w += o.w;
      }
      *reinterpret_cast<float4*>(dst) = r;
    } else {
      const float t[4] = {r.x, r.y, r.z, r.w};
      for (int j = 0; j < 4 && i4 + j < n; ++j) dst[j] = accumulate ? dst[j] + t[j] : t[j];
    }
  }
}

inline void launch_wgrad_reduce(const float* ws, float* dw, long long n, int slices, cudaStream_t st, float* dw2 = nullptr,
                                long long n_first = -1, int accumulate = 0) {
  const unsigned blocks = (unsigned)((n / 4 + 32) / 32);
  if (n_first < 0 || !dw2) { n_first = n; dw2 = dw; }
  wgrad_reduce_kernel<<<blocks, dim3(32, 8), 0, st>>>(ws, dw, n, slices, dw2, n_first, accumulate);
}

struct WgradPlan {
  WgradParams p;
  size_t ws_bytes;
};

// shared planning of the decomposition (also used by the workspace-size query)
int plan_wgrad(WgradPlan& plan, int N, int H, int W, int Cin, int Cout, int R, int S, int stride, int pad, int dil,
               int num_ctas) {
  WgradParams& p = plan.p;
  int Ho, Wo;
  if (!hb::window_out(H, R, stride, pad, dil, Ho) || !hb::window_out(W, S, stride, pad, dil, Wo))
    return (int)cudaErrorInvalidValue;
  const long long m_ll = (long long)N * Ho * Wo;
  if (m_ll > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
  p.m_total = (int)m_ll; p.Ho = Ho; p.Wo = Wo; p.stride = stride; p.pad = pad; p.dil = dil;
  p.R = R; p.S = S; p.Cin = Cin; p.Cout = Cout;
  const int RS = R * S;
  int ci_tile = Cin;
  if (Cin > 128) {
    ci_tile = 128;
    if (Cin % 128 != 0 && Cin % 64 == 0) ci_tile = 64;
  }
  p.ci_tile = ci_tile;
  p.ci_chunks = (ci_tile + 63) / 64;
  p.taps_per_group = 1;
  p.stage_bytes = kABytes + p.ci_chunks * kChunkBytes;
  p.stages = (200 * 1024) / p.stage_bytes;
  if (p.stages > 6) p.stages = 6;
  p.num_tap_groups = (RS + p.taps_per_group - 1) / p.taps_per_group;
  p.num_co_tiles = (Cout + 127) / 128;
  p.num_ci_tiles = (Cin + ci_tile - 1) / ci_tile;
  p.kblocks_total = (p.m_total + kBKpix - 1) / kBKpix;
  const int base_units = p.num_co_tiles * p.num_ci_tiles * p.num_tap_groups;
  const int ctas = num_ctas > 0 ? num_ctas : HB_NUM_SMS;
  int k_splits = (2 * ctas + base_units - 1) / base_units;   // aim at ~2 units per CTA
  if (base_units >= ctas) k_splits = 1;
  const int max_splits = (p.kblocks_total + 7) / 8;          // at least 8 K blocks (512 pixels) per unit
  if (k_splits > max_splits) k_splits = max_splits;
  if (k_splits < 1) k_splits = 1;
  p.k_splits = k_splits;
  p.dw_elems = (long long)Cout * RS * Cin;
  plan.ws_bytes = k_splits > 1 ? (size_t)k_splits * p.dw_elems * sizeof(float) : 0;
  return 0;
}

// Regroups the planned one-tap units into work items of up to `taps` taps of the same (co tile, ci tile, pixel range)
// and sizes the shared-memory ring for their stages. k_splits, the workspace and every unit's result stay as planned.
void group_taps(WgradParams& p, int taps) {
  p.taps_per_group = taps;
  p.num_tap_groups = (p.R * p.S + taps - 1) / taps;
  p.stage_bytes = kABytes + taps * p.ci_chunks * kChunkBytes;
  p.stages = min(6, (200 * 1024) / p.stage_bytes);
}

// Most taps a work item may hold: kMaxTaps, or HB_WGRAD_TAPS_PER_UNIT (1 .. kMaxTaps; 1 runs one tap per unit) so that
// executions can be compared within one build. dW is the same bits for every value.
int max_taps_per_unit() {
  const char* v = getenv("HB_WGRAD_TAPS_PER_UNIT");
  const int n = v ? atoi(v) : kMaxTaps;
  return n < 1 ? 1 : (n > kMaxTaps ? kMaxTaps : n);
}

}  // namespace

extern "C" {

// Bytes of fp32 scratch hb_conv2d_wgrad_bf16 wants for this shape (0 when a single pixel range is used). With a
// workspace the per-range partial sums are written with plain stores and reduced in a fixed order (deterministic);
// without one they are accumulated with fp32 atomics.
size_t hb_conv2d_wgrad_workspace_bytes(int N, int H, int W, int Cin, int Cout, int R, int S, int stride, int pad, int dil,
                                       int num_ctas) {
  WgradPlan plan{};
  if (plan_wgrad(plan, N, H, W, Cin, Cout, R, S, stride, pad, dil, num_ctas)) return 0;
  const size_t rows = hb_wgrad_rows_workspace_bytes(N, H, W, Cin, Cout, R, S, stride, pad, dil, num_ctas, 0);
  return rows > plan.ws_bytes ? rows : plan.ws_bytes;
}

// dW (fp32, [Cout,R,S,Cin]) = wgrad(x [N,H,W,Cin] bf16, dy [N,Ho,Wo,Cout] bf16). Overwrites dW.
// Requirements: Cin % 8 == 0, Cout % 8 == 0, 16-byte aligned pointers.
static int wgrad_impl(const void* x, const void* dy, float* dw, float* workspace, size_t workspace_bytes, int N, int H,
                      int W, int Cin, int Cout, int R, int S, int stride, int pad, int dil, int num_ctas, void* stream,
                      int accumulate) {
  if (Cin % 8 != 0 || Cout % 8 != 0) return (int)cudaErrorInvalidValue;
  if (!hb::aligned16(x) || !hb::aligned16(dy) || !hb::aligned16(dw)) return (int)cudaErrorMisalignedAddress;
  cudaStream_t st = (cudaStream_t)stream;
  static const bool rows_enabled = getenv("HB_DISABLE_WGRAD_ROWS") == nullptr;
  if (rows_enabled && R == 3 && S == 3 && stride == 1 && pad == 1 && dil == 1 && workspace && hb::aligned16(workspace)) {
    int slices = 0;
    const int rc = hb_wgrad_rows_try(x, dy, nullptr, workspace, workspace_bytes, N, H, W, Cin, Cout, num_ctas, st, &slices);
    if (rc == 0) {
      const long long n = (long long)Cout * 9 * Cin;
      launch_wgrad_reduce(workspace, dw, n, slices, st, nullptr, -1, accumulate);
      HB_LAUNCH_CHECK();
      return 0;
    }
    if (rc != (int)cudaErrorNotSupported) return rc;
  }
  WgradPlan plan{};
  if (int rc = plan_wgrad(plan, N, H, W, Cin, Cout, R, S, stride, pad, dil, num_ctas)) return rc;
  WgradParams& p = plan.p;
  // accumulation happens in the fixed-order reduction kernel: it needs the workspace path (more than one pixel range)
  if (accumulate && !(p.k_splits > 1 && workspace && workspace_bytes >= plan.ws_bytes && hb::aligned16(workspace)))
    return (int)cudaErrorNotSupported;
  const int RS = R * S;
  const int k_splits = p.k_splits;
  static const int max_taps = max_taps_per_unit();
  group_taps(p, RS < max_taps ? RS : max_taps);
  const int base_units = p.num_co_tiles * p.num_ci_tiles * p.num_tap_groups;
  const int ctas = num_ctas > 0 ? num_ctas : HB_NUM_SMS;
  p.dw = dw;
  p.ws = workspace;
  if (k_splits == 1) {
    p.use_atomics = 0;
  } else if (workspace && workspace_bytes >= plan.ws_bytes && hb::aligned16(workspace)) {
    p.use_atomics = 2;
  } else {
    p.use_atomics = 1;
    cudaError_t e = cudaMemsetAsync(dw, 0, (size_t)Cout * RS * Cin * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
  }

  CUtensorMap tmDY, tmX;
  if (int rc = tmap::encode_matrix(&tmDY, dy, p.m_total, Cout, kBKpix)) return rc;
  if (int rc = tmap::encode_im2col_bf16(&tmX, x, N, H, W, Cin, pad, pad, R, S, dil, stride, 64, kBKpix,
                                        CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  const size_t smem_bytes = (size_t)p.stages * p.stage_bytes + 2 * p.stages * sizeof(uint64_t) + 1024;
  const int num_units = base_units * k_splits;
  int grid = ctas < num_units ? ctas : num_units;
  // one instantiation per Cin tile width (rounded up to 16) and taps per work item
  const cudaError_t e = dispatch_width<16, 128>((p.ci_tile + 15) & ~15, [&](auto ciw) {
    return dispatch_width<1, kMaxTaps>(p.taps_per_group, [&](auto taps) {
      return launch<conv_wgrad_kernel<decltype(ciw)::value, decltype(taps)::value>>(grid, smem_bytes, st, tmDY, tmX, p);
    });
  });
  if (e != cudaSuccess) return (int)e;
  if (p.use_atomics == 2) {
    const long long n = p.dw_elems;
    launch_wgrad_reduce(workspace, dw, n, k_splits, st, nullptr, -1, accumulate);
    HB_LAUNCH_CHECK();
  }
  return 0;
}

int hb_conv2d_wgrad_bf16(const void* x, const void* dy, float* dw, float* workspace, size_t workspace_bytes, int N, int H,
                         int W, int Cin, int Cout, int R, int S, int stride, int pad, int dil, int num_ctas, void* stream) {
  return wgrad_impl(x, dy, dw, workspace, workspace_bytes, N, H, W, Cin, Cout, R, S, stride, pad, dil, num_ctas, stream, 0);
}

// dW += wgrad(x, dy): the fixed-order reduction adds onto the existing contents of dw (e.g. the parameter's .grad view in
// the flat gradient bucket). Returns cudaErrorNotSupported (801) without touching dw when the shape runs as a single
// pixel range (no reduction pass to fold the addition into): compute into a scratch tensor and add then.
int hb_conv2d_wgrad_acc_bf16(const void* x, const void* dy, float* dw, float* workspace, size_t workspace_bytes, int N, int H,
                             int W, int Cin, int Cout, int R, int S, int stride, int pad, int dil, int num_ctas,
                             void* stream) {
  return wgrad_impl(x, dy, dw, workspace, workspace_bytes, N, H, W, Cin, Cout, R, S, stride, pad, dil, num_ctas, stream, 1);
}

// Both weight gradients of a stride-1 RepVGG block (3x3 pad-1 branch and 1x1 branch over the same input,
// models/classification/repvgg.py:55-73) in one pass over x: dw = [dW3 (Cout,3,3,Cin) | dW1 (Cout,Cin)] fp32, overwritten.
// workspace: hb_repvgg_wgrad_workspace_bytes(...) bytes; a size of 0 means the shape does not fit the row-window scheme
// (call hb_conv2d_wgrad_bf16 twice then); hb_repvgg_wgrad_bf16 returns cudaErrorNotSupported in that case.
size_t hb_repvgg_wgrad_workspace_bytes(int N, int H, int W, int Cin, int Cout, int num_ctas) {
  return hb_wgrad_rows_workspace_bytes(N, H, W, Cin, Cout, 3, 3, 1, 1, 1, num_ctas, 1);
}

static int repvgg_wgrad_impl(const void* x, const void* dy3, const void* dy1, float* dw, float* dw1, float* workspace,
                             size_t workspace_bytes, int N, int H, int W, int Cin, int Cout, int num_ctas, void* stream,
                             int accumulate) {
  if (Cin % 8 != 0 || Cout % 8 != 0) return (int)cudaErrorInvalidValue;
  if (!hb::aligned16(x) || !hb::aligned16(dy3) || !hb::aligned16(dy1) || !hb::aligned16(dw) || !hb::aligned16(workspace) ||
      !hb::aligned16(dw1))
    return (int)cudaErrorMisalignedAddress;
  cudaStream_t st = (cudaStream_t)stream;
  int slices = 0;
  if (int rc = hb_wgrad_rows_try(x, dy3, dy1, workspace, workspace_bytes, N, H, W, Cin, Cout, num_ctas, st, &slices))
    return rc;
  const long long n = (long long)Cout * 10 * Cin;
  launch_wgrad_reduce(workspace, dw, n, slices, st, dw1, dw1 ? (long long)Cout * 9 * Cin : -1, accumulate);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_repvgg_wgrad_bf16(const void* x, const void* dy3, const void* dy1, float* dw, float* workspace, size_t workspace_bytes,
                         int N, int H, int W, int Cin, int Cout, int num_ctas, void* stream) {
  return repvgg_wgrad_impl(x, dy3, dy1, dw, nullptr, workspace, workspace_bytes, N, H, W, Cin, Cout, num_ctas, stream, 0);
}

// dW3 [Cout,3,3,Cin] += ..., dW1 [Cout,Cin] += ...: the two gradients ADDED to separate destination buffers (the .grad
// storage of the two branch filters), one pass over x, one reduction launch.
int hb_repvgg_wgrad_acc_bf16(const void* x, const void* dy3, const void* dy1, float* dw3, float* dw1, float* workspace,
                             size_t workspace_bytes, int N, int H, int W, int Cin, int Cout, int num_ctas, void* stream) {
  if (!dw1) return (int)cudaErrorInvalidValue;
  return repvgg_wgrad_impl(x, dy3, dy1, dw3, dw1, workspace, workspace_bytes, N, H, W, Cin, Cout, num_ctas, stream, 1);
}

}  // extern "C"
