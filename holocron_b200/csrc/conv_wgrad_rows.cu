// Weight gradient of a stride-1 3x3 convolution with few to moderately many channels - the HBM / L2-bound layers - by the
// same "row window" scheme as conv_rows.cu:
//
//   dW[co, r, s, ci] = sum_{n,p,q} dY[n,p,q,co] * X[n,p+r-1,q+s-1,ci]
//
// Per tile (TRO output rows of one image) ONE tiled TMA load brings the TRO+2 input rows (pitch Wp = W+2 pixels, zero
// halo by out-of-bounds fill) and one brings the TRO rows of dY with the SAME pitch (its 2 extra columns per row are
// out-of-bounds zeros), so for tap (r, s) the reduction over pixels is a plain dot product between the dY buffer and the
// X buffer shifted by (r*Wp + s) pixel rows. Both operands are MN-major (pixel index = K): the X window is the A operand
// (M = 64 input channels), dY the B operand (N = output channels of the group).
// Tap slots: the nine taps, plus, for RepVGG blocks (has_b1), the 1x1 branch's weight gradient
// dW1[co, ci] = sum dY1[n,p,q,co] * X[n,p,q,ci], which reads the same X rows through the centre-tap window against a
// second dY buffer. Each consumer warpgroup keeps TPW slots (TPW * NC / 2 <= 64 fp32 registers per thread) for ALL tiles
// of the CTA; there is a single epilogue per CTA that writes a partial dW, reduced afterwards in a fixed order
// (deterministic). Channels and slots beyond one CTA's registers are split into (64-input-channel, <= 64-output-channel,
// slot range) groups; the CTAs of a group share the tiles between them, each group owns a disjoint part of dW.
// The generic kernel (conv_wgrad.cu) re-reads X nine times from L2 (one im2col load per tap).
#include "conv_common.cuh"

namespace {

using namespace tc;
using namespace conv;

struct WRowsParams {
  int N, H, W, Cin, Cout;
  int Wp, TRO, KS;       // smem row pitch, output rows per tile, 16-pixel k-steps per tile
  int n_cig, n_cog, n_sg, ngroups;   // groups of 64 input channels x groups of co_group output channels x slot ranges
  int co_group;          // output channels per group (NC: 16, 32, 48 or 64)
  int tpw;               // tap slots per consumer warpgroup
  int nslots;            // 9, or 10 with the 1x1 branch
  int tiles_per_img, num_tiles;
  int xbuf_bytes, ybuf_bytes, stage_bytes;
  int has_b1;            // 1: also accumulate the 1x1 branch (slot 9, second dY source)
  float* ws;             // [members][dw_elems (+ Cout*Cin)] partial sums
  long long dw_elems;    // Cout*9*Cin
  long long slice_elems; // dw_elems + (has_b1 ? Cout*Cin : 0)
};

// The MMAs of one tile for the first NT of a warpgroup's TPW tap slots (the others lie past nslots): one commit group
// per 16-pixel k-step with one wgmma per slot, so every fence -> commit region is straight-line. Each slot's accumulator
// still takes its k-steps in order. dhi: descriptor high word; `any`: the accumulators already hold earlier tiles.
template <int NC, int NT, int TPW>
__device__ __forceinline__ void wrows_tile_mma(float (&acc)[TPW][NC / 2], const WRowsParams& p, int slot0, uint32_t sx,
                                               uint32_t sy, uint32_t dhi, bool any) {
  static_assert(NT <= TPW, "slot count");
  if constexpr (NT > 0) {
    uint32_t a_lo[NT], b_lo[NT];
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      const int slot = slot0 + t;
      // slot < 9: tap window (r, s) against dY; slot 9: centre window against dY1
      const int off = slot < 9 ? (slot / 3) * p.Wp + (slot % 3) : p.Wp + 1;
      a_lo[t] = desc_lo(sx + off * 128, 16);
      b_lo[t] = desc_lo(slot < 9 ? sy : sy + p.ybuf_bytes, 16);
    }
    for (int k = 0; k < p.KS; ++k) {
      const uint32_t sc = (any || k > 0) ? 1u : 0u;
      const uint32_t kofs = (uint32_t)k * (2048 >> 4);
      wgmma_fence();
#pragma unroll
      for (int t = 0; t < NT; ++t)
        wgmma<NC, 1, 1>(acc[t], make_desc(a_lo[t] + kofs, dhi), make_desc(b_lo[t] + kofs, dhi), sc);
      wgmma_commit();
    }
  }
}

// Picks the instantiation for the run-time number of active slots nt (0 .. TPW).
template <int NC, int NT, int TPW>
__device__ __forceinline__ void wrows_tile_mma_n(int nt, float (&acc)[TPW][NC / 2], const WRowsParams& p, int slot0,
                                                 uint32_t sx, uint32_t sy, uint32_t dhi, bool any) {
  if constexpr (NT > 0) {
    if (nt < NT) {
      wrows_tile_mma_n<NC, NT - 1, TPW>(nt, acc, p, slot0, sx, sy, dhi, any);
      return;
    }
  }
  wrows_tile_mma<NC, NT, TPW>(acc, p, slot0, sx, sy, dhi, any);
}

template <int NC>
__global__ void __launch_bounds__(kThreads, 1)
conv_wgrad_rows_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmDY,
                       const __grid_constant__ CUtensorMap tmDY1, const WRowsParams p) {
  constexpr int TPW = 128 / NC > 8 ? 8 : 128 / NC;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)2 * p.stage_bytes);
  uint64_t* full_bar = bars;       // [2]
  uint64_t* empty_bar = bars + 2;  // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // zero both stages once: rows the TMA boxes never write (tails read by the shifted windows / the rounded-up K range)
  // must be finite zeros, otherwise stale NaN bit patterns times the zero rows of dY would poison the sums
  for (int i = threadIdx.x; i < 2 * p.stage_bytes / 16; i += kThreads)
    reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmX);
    prefetch_tmap(&tmDY);
    for (int i = 0; i < 2; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kConsumers / 32); }
    fence_barrier_init();
  }
  fence_proxy_async();   // generic-proxy zero fill ordered before the async-proxy (TMA / MMA) accesses
  __syncthreads();
  const int group = blockIdx.x % p.ngroups, member = blockIdx.x / p.ngroups, members = gridDim.x / p.ngroups;
  const int ci0 = (group % p.n_cig) * 64, co0 = ((group / p.n_cig) % p.n_cog) * p.co_group;
  const int sg = group / (p.n_cig * p.n_cog);

  if (warp < 4) {
    if (warp == 0 && lane == 0) {
      const uint32_t tx = (uint32_t)((p.TRO + 2) * p.Wp * 128 + (1 + p.has_b1) * p.TRO * p.Wp * 128);
      if (p.has_b1) prefetch_tmap(&tmDY1);
      int it = 0;
      for (int tile = member; tile < p.num_tiles; tile += members, ++it) {
        const int n = tile / p.tiles_per_img, p0 = (tile % p.tiles_per_img) * p.TRO;
        const Ring ring = Ring::at(it, 2);
        uint64_t* bar = &full_bar[ring.stage];
        mbar_wait(&empty_bar[ring.stage], ring.phase ^ 1);
        mbar_arrive_expect_tx(bar, tx);
        uint8_t* sx = smem + (size_t)ring.stage * p.stage_bytes;
        tma_load_4d(&tmX, bar, sx, ci0, -1, p0 - 1, n);
        tma_load_4d(&tmDY, bar, sx + p.xbuf_bytes, co0, 0, p0, n);
        if (p.has_b1) tma_load_4d(&tmDY1, bar, sx + p.xbuf_bytes + p.ybuf_bytes, co0, 0, p0, n);
      }
    }
    return;
  }

  // ================= consumers: warpgroup wg owns slots sg*2*TPW + wg*TPW + [0, TPW) =================
  const int et = threadIdx.x - 128;
  const int wg = et >> 7;
  const int slot0 = sg * 2 * TPW + wg * TPW;
  const uint32_t dhi = desc_hi(1024);
  const int nt = max(0, min(TPW, p.nslots - slot0));   // slots of this warpgroup below nslots
  float acc[TPW][NC / 2];
  bool any = false;
  int it = 0;
  for (int tile = member; tile < p.num_tiles; tile += members, ++it) {
    const Ring ring = Ring::at(it, 2);
    mbar_wait(&full_bar[ring.stage], ring.phase);
    const uint32_t sx = smem_u32(smem + (size_t)ring.stage * p.stage_bytes);
    const uint32_t sy = sx + p.xbuf_bytes;
    wrows_tile_mma_n<NC, TPW, TPW>(nt, acc, p, slot0, sx, sy, dhi, any);
    wgmma_wait<0>();
#pragma unroll
    for (int t = 0; t < TPW; ++t) fence_regs(acc[t]);
    any = true;
    if (lane == 0) mbar_arrive(&empty_bar[ring.stage]);
  }

  // ================= single epilogue per CTA =================
  const bool has_work = member < p.num_tiles;
  float* out = p.ws + (size_t)member * p.slice_elems;
  const int frow = frag_row(et & 127), fcol = frag_col(et & 127);
#pragma unroll
  for (int t = 0; t < TPW; ++t) {
    const int slot = slot0 + t;
    if (slot >= p.nslots) break;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int ci = ci0 + frow + 8 * h;
      if (ci >= p.Cin) continue;
#pragma unroll
      for (int j = 0; j < NC / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 8 * j + fcol + e;
          const int co = co0 + c;
          if (c >= p.co_group || co >= p.Cout) continue;
          const float v = has_work ? acc[t][4 * j + 2 * h + e] : 0.f;
          if (slot < 9) out[((size_t)co * 9 + slot) * p.Cin + ci] = v;
          else out[p.dw_elems + (size_t)co * p.Cin + ci] = v;   // dW1 [Cout][Cin]
        }
      }
    }
  }
}

struct WRowsPlan { WRowsParams p; int grid, members; size_t smem; };

bool plan_wrows(WRowsPlan& pl, int N, int H, int W, int Cin, int Cout, int num_ctas, int has_b1 = 0) {
  if (Cin % 8 != 0 || Cout % 8 != 0 || W < 8 || W + 2 > 128) return false;
  WRowsParams& p = pl.p;
  p.N = N; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout;
  p.Wp = W + 2;
  p.n_cig = (Cin + 63) / 64;
  p.has_b1 = has_b1;
  p.nslots = 9 + has_b1;
  p.n_cog = (Cout + 63) / 64;
  p.co_group = (((Cout + p.n_cog - 1) / p.n_cog) + 15) & ~15;
  p.tpw = 128 / p.co_group > 8 ? 8 : 128 / p.co_group;
  p.n_sg = (p.nslots + 2 * p.tpw - 1) / (2 * p.tpw);
  p.ngroups = p.n_cig * p.n_cog * p.n_sg;
  if (p.ngroups > 32) return false;   // more groups re-read X too often: the generic kernel is the better choice
  int tro = H < 16 ? H : 16;
  for (; tro >= 1; --tro) {
    const int ks = (tro * p.Wp + 15) / 16;
    // X buffer: the last window (offset 2*Wp+2) reads ks*16 rows
    const int xrows = 2 * p.Wp + 2 + ks * 16;
    const int xbytes = ((xrows > (tro + 2) * p.Wp ? xrows : (tro + 2) * p.Wp) * 128 + 1023) & ~1023;
    const int ybytes = ((ks * 16) * 128 + 1023) & ~1023;
    if (2 * (xbytes + (1 + has_b1) * ybytes) <= 220 * 1024) {
      p.TRO = tro; p.KS = ks; p.xbuf_bytes = xbytes; p.ybuf_bytes = ybytes;
      p.stage_bytes = xbytes + (1 + has_b1) * ybytes;
      break;
    }
  }
  if (tro < 1) return false;
  p.tiles_per_img = (H + p.TRO - 1) / p.TRO;
  p.num_tiles = N * p.tiles_per_img;
  p.dw_elems = (long long)Cout * 9 * Cin;
  p.slice_elems = p.dw_elems + (has_b1 ? (long long)Cout * Cin : 0);
  const int ctas = num_ctas > 0 ? num_ctas : HB_NUM_SMS;
  int members = ctas / p.ngroups;
  if (members > p.num_tiles) members = p.num_tiles;
  if (members < 1) return false;
  pl.members = members;
  pl.grid = members * p.ngroups;
  pl.smem = (size_t)2 * p.stage_bytes + 64 + 1024;
  return true;
}

}  // namespace

// workspace bytes wanted by the row-window variant (0 = shape not eligible)
size_t hb_wgrad_rows_workspace_bytes(int N, int H, int W, int Cin, int Cout, int R, int S, int stride, int pad, int dil,
                                     int num_ctas, int has_b1) {
  if (R != 3 || S != 3 || stride != 1 || pad != 1 || dil != 1) return 0;
  WRowsPlan pl{};
  if (!plan_wrows(pl, N, H, W, Cin, Cout, num_ctas, has_b1)) return 0;
  return (size_t)pl.members * pl.p.slice_elems * sizeof(float);
}

// Called from the weight-gradient entry points of conv_wgrad.cu (declared in conv_common.cuh).
int hb_wgrad_rows_try(const void* x, const void* dy, const void* dy1, float* ws, size_t ws_bytes, int N, int H, int W, int Cin,
                      int Cout, int num_ctas, cudaStream_t stream, int* slices_out) {
  constexpr int kNo = (int)cudaErrorNotSupported;
  WRowsPlan pl{};
  const int has_b1 = dy1 != nullptr;
  if (!plan_wrows(pl, N, H, W, Cin, Cout, num_ctas, has_b1)) return kNo;
  WRowsParams& p = pl.p;
  if (!ws || ws_bytes < (size_t)pl.members * p.slice_elems * sizeof(float)) return kNo;
  p.ws = ws;
  CUtensorMap tmX, tmDY, tmDY1;
  if (tmap::encode_nhwc_box(&tmX, x, N, H, W, Cin, p.Wp, p.TRO + 2)) return kNo;
  if (tmap::encode_nhwc_box(&tmDY, dy, N, H, W, Cout, p.Wp, p.TRO)) return kNo;
  if (tmap::encode_nhwc_box(&tmDY1, has_b1 ? dy1 : dy, N, H, W, Cout, p.Wp, p.TRO)) return kNo;
  if (pl.smem > 227 * 1024) return kNo;
  *slices_out = pl.members;
  // one instantiation per output-channel group width
  return (int)dispatch_width<16, 64>(p.co_group, [&](auto nc) {
    return launch<conv_wgrad_rows_kernel<decltype(nc)::value>>(pl.grid, pl.smem, stream, tmX, tmDY, tmDY1, p);
  });
}
