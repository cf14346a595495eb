// Implicit-GEMM 2-D convolution (forward; also the data-gradient pass with transformed weights) on
// the sm_90a tensor cores: NHWC bf16 activations, KRSC bf16 filters, fp32 accumulation in registers (wgmma).
//
// GEMM view:  Y[m, co] = sum_{r,s,ci} X[pix(m) + (r,s), ci] * Wt[co, r, s, ci]
//   M = N*Ho*Wo output pixels (tile 128 = two 64-row warpgroup MMAs), N = Cout (tile BN <= 256),
//   K = R*S*Cin walked tap by tap in 64-channel blocks.
// Replaces the cuDNN calls behind nn.Conv2d in holocron.models.utils.conv_sequence
// (reference holocron/models/utils.py:28-86) and RepBlock (models/classification/repvgg.py:55-73).
//
// Pipeline (one persistent CTA per SM, 384 threads; the producer warpgroup gives registers to the consumers with
// setmaxnreg: 40 + 2 x 232 per thread, so that a consumer thread can hold 128 fp32 accumulators of a 256-column tile):
//   warpgroup 0   TMA producer (one thread): im2col-mode loads of the activation tile (hardware handles padding,
//                 stride, row/image wrap; out-of-range channels are zero-filled) + tiled loads of the filter slab,
//                 both landing 128B-swizzled in a multi-stage smem ring (mbarrier complete_tx).
//   warpgroups 1-2  consumers: each issues wgmma m64nBNk16 for its 64 rows of the 128-row tile (4 per 64-channel
//                 block), keeps one block in flight while it releases the previous stage, then runs the epilogue
//                 of the tile: bias / activation / patch normalisation from the accumulator registers into a bf16
//                 staging tile in shared memory (padded rows, conflict-free), written out with fully coalesced
//                 128-bit stores (+ residual add in that pass). The producer meanwhile fills the ring for the
//                 next tile.
#include <stdlib.h>
#include "conv_common.cuh"
#include "holocron_b200.h"

namespace {

using namespace tc;
using namespace conv;

constexpr int kBM = 128;          // output pixels per tile
constexpr int kBK = 64;           // channels per K block (one 128-byte swizzle row)
constexpr int kMmaK = 16;         // K per wgmma for 16-bit inputs
constexpr int kProducerRegs = 40;   // per thread after setmaxnreg: 128 x (40 + 2 x 232) = 64 512 <= 64 K registers
constexpr int kConsumerRegs = 232;
constexpr int kABytes = kBM * kBK * 2;  // 16 KiB
constexpr int kSmemMax = 227 * 1024;    // dynamic shared memory per CTA on sm_90

struct FpropParams {
  int m_total;      // N*Ho*Wo
  int Ho, Wo;
  int stride, pad_h, pad_w, dil;
  int R, S;
  int Cin, Cout;
  int num_m_tiles, num_n_tiles;
  int cblocks;      // ceil(Cin / 64)
  int ksteps_last;  // 16-channel MMA steps of the last channel block (Cin = 48 -> 3 instead of 4 zero-padded ones)
  // extra K blocks issued after the R*S*cblocks main ones:
  //   e_mode 1: a second source xe [M, Ce] (rows = the output rows) with filter we [Cout,1,1,Ce] accumulated into the
  //             SAME accumulator (K extension: dX = dgrad3x3(dY3) + dgrad1x1(dY1) in one kernel);
  //   e_mode 2: the centre tap of the main source once more with a second filter w2 [Cout,1,1,Cin] into a SECOND
  //             accumulator (dual output: y = conv RxS, y2 = conv 1x1 of the same input, same stride - RepVGG forward).
  int e_mode, e_cblocks, e_ksteps_last;
  int nout;         // 1, or 2 in dual mode
  int stages;
  int b_stage_bytes;  // BN*128 rounded up to 1024 (BN: the Cout tile, a template parameter of the kernel)
  int out_pitch;      // bytes per row of the smem output staging tile (min(BN, 64)*2 + 16)
  int a_mode;         // 0: plain 2-D [M, C] matrix (1x1 s1 p0), 1: im2col
  int act;            // 0 none, 1 relu
  __nv_bfloat16* y;
  __nv_bfloat16* y2;              // dual mode: second output (same addressing as y)
  // optional per-channel statistics of the bf16 OUTPUT (what the BatchNorm that follows normalises), in the slot format
  // of conv_common.cuh, slot = (blockIdx.x / num_n_tiles) * 2 + consumer warpgroup
  float* stats;
  float* stats2;
  const float* bias;              // [Cout] or null
  const __nv_bfloat16* residual;  // [M, Cout] or null (same addressing as y)
  // patch normalisation in the epilogue (NormConv2d, reference nn/functional.py:322-413): with the per-patch statistics of
  // the im2col rows, y = rstd[m] * (acc - mean[m] * wsum[co]) (+ bias) == sum_k ((patch_k - mean) * rstd) * w[co, k]
  const float* norm_mean;         // [M] or null
  const float* norm_rstd;         // [M]
  const float* norm_wsum;         // [Cout] = sum over (r, s, ci) of the bf16 filter
  // output addressing: dense rows (scatter == 0) or output pixel (n, i, j) of the Ho x Wo grid written to pixel
  // (i*o_step + o_a, j*o_step + o_b) of an OH x OW image (the parity classes of a strided data gradient)
  int scatter, OH, OW, o_step, o_a, o_b;
};

// kStats: the epilogue also accumulates the output-column statistics (separate instantiation: the plain kernel carries
// neither the extra registers nor the extra shared-memory pass in its instruction stream).
// BN: the Cout tile (a multiple of 16 up to 256, at most 64 in dual mode), the N of every wgmma.
template <bool kStats, int BN>
__global__ void __launch_bounds__(kThreads, 1)
conv_fprop_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2, const FpropParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [stages][A | B], staging tile + row offset table, then barriers
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int stage_bytes = kABytes + p.b_stage_bytes;
  uint8_t* sout = smem + (size_t)p.stages * stage_bytes;
  const size_t sout_bytes = (((size_t)kBM * p.out_pitch + 15) & ~(size_t)15) + kBM * sizeof(long long);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sout + sout_bytes);
  uint64_t* empty_bar = full_bar + p.stages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    if (p.e_mode) { prefetch_tmap(&tmB2); if (p.e_mode == 1) prefetch_tmap(&tmA2); }
    for (int i = 0; i < p.stages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kConsumers / 32); }
    fence_barrier_init();
  }
  __syncthreads();

  // Tile walk: CTA b always works on Cout tile  b % num_n_tiles  (gridDim.x is a multiple of num_n_tiles) and takes the
  // pixel tiles  b / num_n_tiles + k * (gridDim.x / num_n_tiles): CTAs that run side by side share their A tile in L2, and
  // the per-CTA column statistics cover a fixed channel range.
  const int n_tile = blockIdx.x % p.num_n_tiles;
  const int m_first = blockIdx.x / p.num_n_tiles, m_step = gridDim.x / p.num_n_tiles;
  const int kblocks = p.R * p.S * p.cblocks;
  const uint32_t tx_bytes = kABytes + BN * 128;

  if (warp < 4) {
    // ================= TMA producer =================
    regs_release<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      Ring ring;
      for (int m_tile = m_first; m_tile < p.num_m_tiles; m_tile += m_step) {
        const int m0 = m_tile * kBM;
        const int q0 = m0 % p.Wo, p0 = (m0 / p.Wo) % p.Ho, n0 = m0 / (p.Wo * p.Ho);
        const int base_w = q0 * p.stride - p.pad_w, base_h = p0 * p.stride - p.pad_h;
        for (int tap = 0; tap < p.R * p.S; ++tap) {
          const int r = tap / p.S, s = tap % p.S;
          for (int cb = 0; cb < p.cblocks; ++cb) {
            uint64_t* bar = &full_bar[ring.stage];
            mbar_wait(&empty_bar[ring.stage], ring.phase ^ 1);
            uint8_t* sa = smem + (size_t)ring.stage * stage_bytes;
            uint8_t* sb = sa + kABytes;
            mbar_arrive_expect_tx(bar, tx_bytes);
            if (p.a_mode == 1)
              tma_load_im2col_4d(&tmA, bar, sa, cb * kBK, base_w, base_h, n0, (uint16_t)(s * p.dil), (uint16_t)(r * p.dil));
            else
              tma_load_2d(&tmA, bar, sa, cb * kBK, m0);
            tma_load_3d(&tmB, bar, sb, cb * kBK, tap, n_tile * BN);
            ring.next(p.stages);
          }
        }
        for (int cb = 0; cb < p.e_cblocks; ++cb) {
          uint64_t* bar = &full_bar[ring.stage];
          mbar_wait(&empty_bar[ring.stage], ring.phase ^ 1);
          uint8_t* sa = smem + (size_t)ring.stage * stage_bytes;
          uint8_t* sb = sa + kABytes;
          mbar_arrive_expect_tx(bar, tx_bytes);
          if (p.e_mode == 1)
            tma_load_2d(&tmA2, bar, sa, cb * kBK, m0);
          else if (p.a_mode == 1)
            tma_load_im2col_4d(&tmA, bar, sa, cb * kBK, base_w, base_h, n0, (uint16_t)((p.S / 2) * p.dil),
                               (uint16_t)((p.R / 2) * p.dil));
          else
            tma_load_2d(&tmA, bar, sa, cb * kBK, m0);
          tma_load_3d(&tmB2, bar, sb, cb * kBK, 0, n_tile * BN);
          ring.next(p.stages);
        }
      }
    }
    return;
  }

  // ================= consumers: MMA + epilogue =================
  regs_acquire<kConsumerRegs>();
  const int et = threadIdx.x - 128;        // 0..255
  const int wg = et >> 7;                  // rows [64*wg, 64*wg + 64) of every tile
  const int wet = et & 127;
  const int frow = 64 * wg + frag_row(wet);   // this thread's first accumulator row (second: +8)
  const int fcol = frag_col(wet);
  const uint32_t dhi = desc_hi(1024);
  const uint32_t a_lo0 = desc_lo(smem_u32(smem), 16) + (uint32_t)wg * ((64 * 128) >> 4);
  const uint32_t stage_lo = (uint32_t)stage_bytes >> 4;
  long long* row_off = reinterpret_cast<long long*>(sout + (((size_t)kBM * p.out_pitch + 15) & ~(size_t)15));
  // column groups of <= 64 columns go through the fixed-size staging tile: gpo groups per output, nout outputs
  const int gpo = (BN + 63) >> 6;
  const int ngroups = p.nout * gpo;
  // column statistics: this thread's running (sum0, sum1, sumsq0, sumsq1) of one column PAIR of each group over a fixed
  // subset of its warpgroup's 64 tile rows, kept in registers across all tiles of the CTA
  float4 st[4];
#pragma unroll
  for (int gi = 0; gi < 4; ++gi) st[gi] = make_float4(0.f, 0.f, 0.f, 0.f);
  const int col_base = n_tile * BN;
  const int ncols_valid = min(BN, p.Cout - col_base);          // multiple of 16
  // accumulator columns: BN, or 2 x BN for the second output of dual mode (only possible for BN <= 64)
  constexpr int kCols = BN <= 64 ? 2 * BN : BN;
  float acc[kCols / 2];
  Ring ring;

  for (int m_tile = m_first; m_tile < p.num_m_tiles; m_tile += m_step) {
    // ---- main loop: one commit group per K block; one block stays in flight while the stage of the previous one
    // is handed back to the producer ----
    int prev = -1;
    auto next_block = [&](uint32_t& a_lo, uint32_t& b_lo) {
      mbar_wait(&full_bar[ring.stage], ring.phase);
      a_lo = a_lo0 + (uint32_t)ring.stage * stage_lo;
      b_lo = desc_lo(smem_u32(smem), 16) + (uint32_t)ring.stage * stage_lo + (kABytes >> 4);
    };
    auto retire_prev = [&]() {
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);   // the MMAs that read stage `prev` are done
      prev = ring.stage;
      ring.next(p.stages);
    };
    for (int kb = 0, cb = 0; kb < kblocks; ++kb) {
      uint32_t a_lo, b_lo;
      next_block(a_lo, b_lo);
      if (++cb == p.cblocks) {
        cb = 0;
        wgmma_group_ks<BN, 0, 0>(p.ksteps_last, acc, a_lo, b_lo, 2, dhi, kb != 0);
      } else {
        wgmma_group<BN, kBK / kMmaK, 0, 0>(acc, a_lo, b_lo, 2, dhi, kb != 0);
      }
      retire_prev();
    }
    // extra K blocks: same accumulator (e_mode 1) or the second accumulator, BN columns further (e_mode 2)
    for (int ecb = 0; ecb < p.e_cblocks; ++ecb) {
      uint32_t a_lo, b_lo;
      next_block(a_lo, b_lo);
      const int ks = (ecb == p.e_cblocks - 1) ? p.e_ksteps_last : kBK / kMmaK;
      if constexpr (BN <= 64) {
        if (p.e_mode == 2) wgmma_group_ks<BN, 0, 0>(ks, acc + BN / 2, a_lo, b_lo, 2, dhi, ecb != 0);
        else wgmma_group_ks<BN, 0, 0>(ks, acc, a_lo, b_lo, 2, dhi, 1u);
      } else {
        wgmma_group_ks<BN, 0, 0>(ks, acc, a_lo, b_lo, 2, dhi, 1u);
      }
      retire_prev();
    }
    wgmma_wait<0>();
    fence_regs(acc);
    if (lane == 0) mbar_arrive(&empty_bar[prev]);

    // ---- epilogue ----
    const int rows_valid = min(kBM, p.m_total - m_tile * kBM);
    float nm[2] = {0.f, 0.f}, nr[2] = {1.f, 1.f};
    if (p.norm_mean) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m_row = m_tile * kBM + frow + 8 * h;
        if (m_row < p.m_total) { nm[h] = __ldg(p.norm_mean + m_row); nr[h] = __ldg(p.norm_rstd + m_row); }
      }
    }
#pragma unroll 1
    for (int gi = 0; gi < ngroups; ++gi) {
      const int o = gi >= gpo ? 1 : 0;                 // output index (dual mode: 0 = RxS conv, 1 = 1x1 conv)
      const int g0 = (gi - o * gpo) * 64;
      const int gw = min(64, BN - g0);
      __nv_bfloat16* yo = o ? p.y2 : p.y;
      const bool first = o == 0;
      const int cs0 = o * BN + g0;                   // first accumulator column of this group
      consumer_sync();   // staging tile free
      if (gi == 0 && et < kBM) {
        // element offset of each output row of the tile (read by every thread in the copy-out below)
        const long long m = (long long)m_tile * kBM + et;
        if (!p.scatter) {
          row_off[et] = m * p.Cout;
        } else {
          const int j = (int)(m % p.Wo), i = (int)((m / p.Wo) % p.Ho), n = (int)(m / ((long long)p.Wo * p.Ho));
          row_off[et] = (((long long)n * p.OH + (long long)i * p.o_step + p.o_a) * p.OW + (long long)j * p.o_step + p.o_b) * p.Cout;
        }
      }
#pragma unroll
      for (int j = 0; j < kCols / 8; ++j) {
        const int cs = 8 * j + fcol;                   // accumulator column of registers 4j .. 4j+3
        if (cs >= cs0 && cs < cs0 + gw) {
          const int cl = cs - cs0;                     // column inside the staged group
          const int col = col_base + g0 + cl;
          const bool ok = col < p.Cout;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
            if (first && p.norm_mean && ok) {
              f0 = nr[h] * (f0 - nm[h] * __ldg(p.norm_wsum + col));
              f1 = nr[h] * (f1 - nm[h] * __ldg(p.norm_wsum + col + 1));
            }
            if (first && p.bias && ok) { f0 += __ldg(p.bias + col); f1 += __ldg(p.bias + col + 1); }
            if (first && p.act == 1 && !p.residual) { f0 = hb::relu_nan(f0); f1 = hb::relu_nan(f1); }
            *reinterpret_cast<__nv_bfloat162*>(sout + (size_t)(frow + 8 * h) * p.out_pitch + cl * 2) =
                __floats2bfloat162_rn(f0, f1);
          }
        }
      }
      consumer_sync();   // staged group visible to both warpgroups
      const int chunks_per_row = gw / 8;
      const int total_chunks = rows_valid * chunks_per_row;
      int r = et / chunks_per_row, c8 = et - r * chunks_per_row;
      const int dr = kConsumers / chunks_per_row, dc = kConsumers - dr * chunks_per_row;
      const __nv_bfloat16* resid = first ? p.residual : nullptr;
      if (!resid) {
        for (int ch = et; ch < total_chunks; ch += kConsumers) {
          if (g0 + c8 * 8 < ncols_valid) {
            const uint4 val = *reinterpret_cast<const uint4*>(sout + (size_t)r * p.out_pitch + c8 * 16);
            *reinterpret_cast<uint4*>(yo + (size_t)row_off[r] + col_base + g0 + c8 * 8) = val;
          }
          r += dr; c8 += dc;
          if (c8 >= chunks_per_row) { c8 -= chunks_per_row; ++r; }
        }
      } else {
        // residual add: the global loads of 4 trips are issued before the first one is consumed (one dependent
        // global load per trip made this pass latency-bound)
        for (int ch = et; ch < total_chunks; ch += 4 * kConsumers) {
          size_t off[4];
          int sidx[4];
          uint4 rv[4];
          bool ok[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            ok[u] = (ch + u * kConsumers < total_chunks) && (g0 + c8 * 8 < ncols_valid);
            sidx[u] = r * p.out_pitch + c8 * 16;
            off[u] = ok[u] ? (size_t)row_off[r] + col_base + g0 + c8 * 8 : 0;
            if (ok[u]) rv[u] = *reinterpret_cast<const uint4*>(resid + off[u]);
            r += dr; c8 += dc;
            if (c8 >= chunks_per_row) { c8 -= chunks_per_row; ++r; }
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            if (!ok[u]) continue;
            uint4 val = *reinterpret_cast<const uint4*>(sout + sidx[u]);
            add_residual16(val, rv[u], p.act == 1);
            *reinterpret_cast<uint4*>(yo + off[u]) = val;
          }
        }
      }
      if (kStats && (o ? (p.stats2 != nullptr) : (p.stats != nullptr))) {
        // per-channel sum / sum of squares of the staged (bf16-rounded) tile: thread = (column pair, row subset of its
        // warpgroup's 64 rows)
        const int npairs = gw >> 1, rgs = 128 / npairs;
        const int rg = wet / npairs, pr = wet - rg * npairs;
        const int row_end = min(64 * wg + 64, rows_valid);
        if (rg < rgs && g0 + pr * 2 < ncols_valid) {
          const uint8_t* sp = sout + pr * 4;
          float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
          for (int rr = 64 * wg + rg; rr < row_end; rr += rgs) accum_pair(s, sp + (size_t)rr * p.out_pitch);
#pragma unroll
          for (int g = 0; g < 4; ++g)
            if (g == gi) { st[g].x += s.x; st[g].y += s.y; st[g].z += s.z; st[g].w += s.w; }
        }
      }
    }
  }
  // ---- statistics: fold the row subsets in a fixed order and write this (CTA, warpgroup)'s partial
  if (kStats && (p.stats || p.stats2)) {
    const int slot = (blockIdx.x / p.num_n_tiles) * 2 + wg;
#pragma unroll
    for (int gi = 0; gi < 4; ++gi) {
      if (gi >= ngroups) break;
      const int o = gi >= gpo ? 1 : 0;
      float* so = o ? p.stats2 : p.stats;
      if (!so) continue;
      const int g0 = (gi - o * gpo) * 64;
      const int gw = min(64, BN - g0);
      const int npairs = gw >> 1, rgs = 128 / npairs;
      consumer_sync();
      float4* scratch = reinterpret_cast<float4*>(sout) + wg * 128;   // [2][128] float4, 4 KB <= staging tile
      scratch[wet] = st[gi];
      consumer_sync();
      if (wet < gw && g0 + wet < ncols_valid)
        store_stats(so, slot, p.Cout, col_base + g0 + wet, fold_stats(scratch, rgs, npairs, wet));
    }
  }
}

struct FpropArgs {
  const void* x; const void* w; void* y; const float* bias; const void* residual;
  int N, H, W, Cin, Cout, R, S, stride;
  int pad_h, pad_w, pad_after_h, pad_after_w, dil, act, num_ctas;
  int Ho, Wo;                      // output grid walked by the GEMM rows
  int scatter, OH, OW, o_step, o_a, o_b;
  // K extension (same accumulator): xe [M, Ce] bf16 rows aligned with the output rows, we [Cout,1,1,Ce]
  const void* xe; const void* we; int Ce;
  // dual output: w2 [Cout,1,1,Cin] applied to the centre tap of x -> y2
  const void* w2; void* y2;
  float* stats; float* stats2; int* stat_slots;
  const float* norm_mean; const float* norm_rstd; const float* norm_wsum;
  cudaStream_t stream;
};

int fprop_launch(const FpropArgs& a) {
  const int Cin = a.Cin, Cout = a.Cout, R = a.R, S = a.S;
  const long long m_total_ll = (long long)a.N * a.Ho * a.Wo;
  if (a.Ho <= 0 || a.Wo <= 0 || m_total_ll <= 0 || m_total_ll > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
  const bool dual = a.w2 != nullptr;
  const bool kext = a.xe != nullptr;
  if (dual && kext) return (int)cudaErrorInvalidValue;
  if (dual && (!a.y2 || a.scatter || !(R & 1) || !(S & 1))) return (int)cudaErrorInvalidValue;
  if (kext && (!a.we || a.Ce % 8 != 0 || a.scatter || !hb::aligned16(a.xe) || !hb::aligned16(a.we)))
    return (int)cudaErrorInvalidValue;
  FpropParams p{};
  p.m_total = (int)m_total_ll;
  p.Ho = a.Ho; p.Wo = a.Wo;
  p.stride = a.stride; p.pad_h = a.pad_h; p.pad_w = a.pad_w; p.dil = a.dil;
  p.R = R; p.S = S; p.Cin = Cin; p.Cout = Cout;
  p.scatter = a.scatter; p.OH = a.OH; p.OW = a.OW; p.o_step = a.o_step; p.o_a = a.o_a; p.o_b = a.o_b;
  p.num_m_tiles = (p.m_total + kBM - 1) / kBM;
  int grid = a.num_ctas > 0 ? a.num_ctas : HB_NUM_SMS;
  if (grid > HB_NUM_SMS * 4) grid = HB_NUM_SMS * 4;
  // Cout tile. Narrow rule: whole Cout up to 128 columns (64 per output in dual mode), else the largest multiple of 16
  // below that limit that divides Cout (falls back to the limit with a masked tail). Wide rule (single output, filters
  // with more than one tap, no output statistics): whole Cout up to 256, else 256 or 192 when it divides Cout. A wide
  // tile multiplies each activation tile it loads into twice the columns. It is only taken while there are still at
  // least as many tiles as CTAs in the grid, so small-M layers keep their parallelism; not for 1x1 filters: their K
  // loop is short next to the epilogue, and on an H100 their wide tiles measured slower than the narrow ones; and not
  // with statistics: each (CTA, warpgroup) slot sums the tiles of its CTA in order, so the Cout tile sets which partial
  // sums the BatchNorm adds up, and the narrow tiles keep those sums, to the bit, as they were.
  const int bn_max = dual ? 64 : 128;
  int BN = Cout;
  if (Cout > bn_max) {
    BN = bn_max;
    for (int c = bn_max; c >= 64; c -= 16) if (Cout % c == 0) { BN = c; break; }
    const int wide = dual || R * S == 1 || a.stats ? 0 : Cout <= 256 ? Cout : Cout % 256 == 0 ? 256 : Cout % 192 == 0 ? 192 : 0;
    if (wide && (long long)p.num_m_tiles * (Cout / wide) >= grid) BN = wide;
  }
  p.nout = dual ? 2 : 1;
  p.num_n_tiles = (Cout + BN - 1) / BN;
  p.cblocks = (Cin + kBK - 1) / kBK;
  p.ksteps_last = ((Cin - (p.cblocks - 1) * kBK) + kMmaK - 1) / kMmaK;
  p.e_mode = kext ? 1 : (dual ? 2 : 0);
  const int ce = kext ? a.Ce : (dual ? Cin : 0);
  p.e_cblocks = (ce + kBK - 1) / kBK;
  p.e_ksteps_last = p.e_cblocks ? ((ce - (p.e_cblocks - 1) * kBK) + kMmaK - 1) / kMmaK : 0;
  p.b_stage_bytes = ((BN * 128) + 1023) & ~1023;
  p.out_pitch = (BN < 64 ? BN : 64) * 2 + 16;
  const int out_bytes = ((((kBM * p.out_pitch + 15) & ~15) + kBM * 8) + 1023) & ~1023;   // staging tile + row offsets
  const int stage_bytes = kABytes + p.b_stage_bytes;
  // as many ring stages as the 227 KiB of dynamic shared memory hold next to the staging tile, the barriers and the
  // 1 KiB alignment slack (BN = 256: 4 stages of 48 KiB)
  int stages = (kSmemMax - 1024 - out_bytes - 2 * 8 * (int)sizeof(uint64_t)) / stage_bytes;
  if (stages > 8) stages = 8;
  if (stages < 2) return (int)cudaErrorInvalidValue;
  p.stages = stages;
  p.a_mode = (R == 1 && S == 1 && a.stride == 1 && a.pad_h == 0 && a.pad_w == 0 && a.pad_after_h == 0 &&
              a.pad_after_w == 0) ? 0 : 1;
  p.act = a.act;
  p.y = (__nv_bfloat16*)a.y;
  p.y2 = (__nv_bfloat16*)a.y2;
  p.stats = a.stats; p.stats2 = dual ? a.stats2 : nullptr;
  p.bias = a.bias;
  p.residual = (const __nv_bfloat16*)a.residual;
  p.norm_mean = a.norm_mean; p.norm_rstd = a.norm_rstd; p.norm_wsum = a.norm_wsum;
  if (p.norm_mean && (!p.norm_rstd || !p.norm_wsum || a.scatter)) return (int)cudaErrorInvalidValue;

  CUtensorMap tmA, tmB, tmA2, tmB2;
  int rc = p.a_mode == 0 ? tmap::encode_matrix(&tmA, a.x, p.m_total, Cin, kBM)
                         : tmap::encode_im2col_bf16(&tmA, a.x, a.N, a.H, a.W, Cin, a.pad_h, a.pad_w, R, S, a.dil,
                                                    a.stride, kBK, kBM, CU_TENSOR_MAP_SWIZZLE_128B, a.pad_after_h,
                                                    a.pad_after_w);
  if (rc) return rc;
  if ((rc = tmap::encode_krsc_slab(&tmB, a.w, Cout, R * S, Cin, BN))) return rc;
  tmA2 = tmA; tmB2 = tmB;   // unused slots alias the main maps (never dereferenced by the kernel)
  if (kext && (rc = tmap::encode_matrix(&tmA2, a.xe, p.m_total, a.Ce, kBM))) return rc;
  if (p.e_mode && (rc = tmap::encode_krsc_slab(&tmB2, kext ? a.we : a.w2, Cout, 1, ce, BN))) return rc;

  const size_t smem_bytes = (size_t)stages * stage_bytes + out_bytes + 2 * stages * sizeof(uint64_t) + 1024;
  // grid: a multiple of num_n_tiles (every CTA keeps one Cout tile), at most one CTA per SM / per tile
  int per_n = grid / p.num_n_tiles;
  if (per_n < 1) per_n = 1;
  if (per_n > p.num_m_tiles) per_n = p.num_m_tiles;
  grid = per_n * p.num_n_tiles;
  if (a.stat_slots) *a.stat_slots = 2 * per_n;
  const bool stats = p.stats || p.stats2;
  // one instantiation per Cout tile width, with and without the statistics epilogue; wide tiles never carry the
  // statistics epilogue (see the Cout tile rule above)
  return (int)dispatch_width<16, 256>(BN, [&](auto bn) {
    constexpr int kBN = decltype(bn)::value;
    if constexpr (kBN > 128) {
      if (stats) return cudaErrorInvalidValue;
      return launch<conv_fprop_kernel<false, kBN>>(grid, smem_bytes, a.stream, tmA, tmB, tmA2, tmB2, p);
    } else {
      return stats ? launch<conv_fprop_kernel<true, kBN>>(grid, smem_bytes, a.stream, tmA, tmB, tmA2, tmB2, p)
                   : launch<conv_fprop_kernel<false, kBN>>(grid, smem_bytes, a.stream, tmA, tmB, tmA2, tmB2, p);
    }
  });
}

}  // namespace

extern "C" {

// Forward convolution, NHWC bf16.  x: [N,H,W,Cin]  w: [Cout,R,S,Cin]  y: [N,Ho,Wo,Cout]
//   bias: fp32 [Cout] or NULL; residual: bf16 [N,Ho,Wo,Cout] or NULL; act: 0 none, 1 relu.
// Requirements: Cin % 8 == 0, Cout % 16 == 0, all pointers 16-byte aligned.
int hb_conv2d_fprop_bf16(const void* x, const void* w, void* y, const float* bias, const void* residual, int N, int H,
                         int W, int Cin, int Cout, int R, int S, int stride, int pad, int dil, int act, int num_ctas,
                         void* stream) {
  hb_conv_args a{};
  a.x = x; a.w = w; a.y = y; a.bias = bias; a.residual = residual;
  a.N = N; a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout; a.R = R; a.S = S; a.stride = stride; a.pad = pad; a.dil = dil;
  a.act = act; a.num_ctas = num_ctas;
  return hb_conv2d_fused_bf16(&a, nullptr, stream);
}

int hb_conv_stat_slots_max(void) { return 2 * HB_NUM_SMS * 4; }

// General form (see include/holocron_b200.h): K extension, dual output and output-column statistics.
int hb_conv2d_fused_bf16(const hb_conv_args* c, int* stat_slots, void* stream) {
  if (!c) return (int)cudaErrorInvalidValue;
  const int N = c->N, H = c->H, W = c->W, Cin = c->Cin, Cout = c->Cout, R = c->R, S = c->S;
  const int stride = c->stride, pad = c->pad, dil = c->dil;
  if (Cin % 8 != 0 || Cout % 16 != 0) return (int)cudaErrorInvalidValue;
  if (!hb::aligned16(c->x) || !hb::aligned16(c->w) || !hb::aligned16(c->y)) return (int)cudaErrorMisalignedAddress;
  if (c->w2 && (!hb::aligned16(c->w2) || !hb::aligned16(c->y2))) return (int)cudaErrorMisalignedAddress;
  int Ho, Wo;
  if (!hb::window_out(H, R, stride, pad, dil, Ho) || !hb::window_out(W, S, stride, pad, dil, Wo))
    return (int)cudaErrorInvalidValue;
  if ((long long)N * Ho * Wo > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
  if (c->w2 && pad != (R / 2) * dil) return (int)cudaErrorInvalidValue;   // centre tap == the 1x1 pad-0 conv's input
  if ((c->stats || c->stats2) && !stat_slots) return (int)cudaErrorInvalidValue;

  if (R == 3 && S == 3 && stride == 1 && pad == 1 && dil == 1 && !c->xe && !c->w2 && !c->norm_mean) {
    static const bool rows_enabled = getenv("HB_DISABLE_CONV_ROWS") == nullptr;
    if (rows_enabled) {
      const int rc = hb_conv_rows_try(c->x, c->w, c->y, c->bias, c->residual, N, H, W, Cin, Cout, c->act, c->num_ctas,
                                      (cudaStream_t)stream, 0, nullptr, nullptr, c->stats, stat_slots);
      if (rc != (int)cudaErrorNotSupported) return rc;
    }
  }
  FpropArgs a{};
  a.x = c->x; a.w = c->w; a.y = c->y; a.bias = c->bias; a.residual = c->residual;
  a.N = N; a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout; a.R = R; a.S = S; a.stride = stride;
  a.pad_h = a.pad_w = a.pad_after_h = a.pad_after_w = pad; a.dil = dil; a.act = c->act; a.num_ctas = c->num_ctas;
  a.Ho = Ho; a.Wo = Wo; a.stream = (cudaStream_t)stream;
  a.xe = c->xe; a.we = c->we; a.Ce = c->Ce; a.w2 = c->w2; a.y2 = c->y2;
  a.stats = c->stats; a.stats2 = c->stats2; a.stat_slots = stat_slots;
  a.norm_mean = c->norm_mean; a.norm_rstd = c->norm_rstd; a.norm_wsum = c->norm_wsum;
  return fprop_launch(a);
}

// Data gradient of a stride-2 3x3 pad-1 convolution WITHOUT zero insertion: the four (row, column) parity classes of dx
// are four small stride-1 correlations over dy (1, 2, 2 and 4 taps), each written straight to its sub-grid of dx:
//   dx[2i+a, 2j+b] = sum_{t,u} dy[i+t, j+u] * wcls_ab[t, u]       t < 1+a, u < 1+b
// 9/4 of the multiply-adds per pixel instead of 9, dy read at its own resolution, no H x W scratch tensors.
//   dy: [N,Ho,Wo,C] bf16; wcls: the class filters from hb_pack_dgrad_s2_weights; dx: [N,H,W,Cd] bf16 (every element written).
//   dy1/wd1 (optional): output gradient and [Cd][C] filter of a parallel 1x1 stride-2 branch (RepVGG), whose data gradient
//   only touches class (0,0); it is written first and the 3x3 class accumulates onto it.
int hb_conv2d_dgrad_s2_bf16(const void* dy, const void* wcls, const void* dy1, const void* wd1, void* dx, int N, int H, int W,
                            int Ho, int Wo, int C, int Cd, int num_ctas, void* stream) {
  if (C % 8 != 0 || Cd % 16 != 0) return (int)cudaErrorInvalidValue;
  if (!hb::aligned16(dy) || !hb::aligned16(wcls) || !hb::aligned16(dx)) return (int)cudaErrorMisalignedAddress;
  if (Ho != (H - 1) / 2 + 1 || Wo != (W - 1) / 2 + 1 || H < 2 || W < 2) return (int)cudaErrorInvalidValue;
  const __nv_bfloat16* wc = (const __nv_bfloat16*)wcls;
  size_t woff = 0;
  for (int a = 0; a < 2; ++a) {
    for (int b = 0; b < 2; ++b) {
      const int Hc = (H - a + 1) / 2, Wc = (W - b + 1) / 2;   // pixels of this parity class
      const int R = 1 + a, S = 1 + b;
      FpropArgs f{};
      f.x = dy; f.w = wc + woff; f.y = dx; f.bias = nullptr; f.residual = nullptr;
      f.N = N; f.H = Ho; f.W = Wo; f.Cin = C; f.Cout = Cd; f.R = R; f.S = S; f.stride = 1;
      f.pad_h = 0; f.pad_w = 0;
      f.pad_after_h = a ? Hc + 1 - Ho : 0;   // 1 when the last odd row reaches dy row Ho (zero), else 0
      f.pad_after_w = b ? Wc + 1 - Wo : 0;
      f.dil = 1; f.act = 0; f.num_ctas = num_ctas;
      f.Ho = Hc; f.Wo = Wc;
      f.scatter = 1; f.OH = H; f.OW = W; f.o_step = 2; f.o_a = a; f.o_b = b;
      f.stream = (cudaStream_t)stream;
      if (a == 0 && b == 0 && dy1 && wd1) {
        FpropArgs g = f;
        g.x = dy1; g.w = wd1;
        if (int rc = fprop_launch(g)) return rc;
        f.residual = dx;   // accumulate onto the 1x1 branch's contribution
      }
      if (Hc > 0 && Wc > 0) {
        if (int rc = fprop_launch(f)) return rc;
      }
      woff += (size_t)Cd * R * S * C;
    }
  }
  return 0;
}

}  // extern "C"
