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
#include "common.cuh"
#include "tc_common.cuh"
#include "tmap.cuh"

namespace {

using namespace tc;

constexpr int kThreads = 384;   // producer warpgroup + 2 consumer warpgroups
constexpr int kConsumers = 256;

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
        const int st = it & 1;
        const int n = tile / p.tiles_per_img, p0 = (tile % p.tiles_per_img) * p.TRO;
        mbar_wait(&empty_bar[st], ((it >> 1) & 1) ^ 1);
        mbar_arrive_expect_tx(&full_bar[st], tx);
        uint8_t* sx = smem + (size_t)st * p.stage_bytes;
        asm volatile(
            "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
            ::"r"(smem_u32(sx)), "l"(reinterpret_cast<uint64_t>(&tmX)), "r"(smem_u32(&full_bar[st])), "r"(ci0), "r"(-1),
              "r"(p0 - 1), "r"(n) : "memory");
        asm volatile(
            "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
            ::"r"(smem_u32(sx + p.xbuf_bytes)), "l"(reinterpret_cast<uint64_t>(&tmDY)),
              "r"(smem_u32(&full_bar[st])), "r"(co0), "r"(0), "r"(p0), "r"(n) : "memory");
        if (p.has_b1)
          asm volatile(
              "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
              ::"r"(smem_u32(sx + p.xbuf_bytes + p.ybuf_bytes)), "l"(reinterpret_cast<uint64_t>(&tmDY1)),
                "r"(smem_u32(&full_bar[st])), "r"(co0), "r"(0), "r"(p0), "r"(n) : "memory");
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
    const int st = it & 1;
    mbar_wait(&full_bar[st], (it >> 1) & 1);
    const uint32_t sx = smem_u32(smem + (size_t)st * p.stage_bytes);
    const uint32_t sy = sx + p.xbuf_bytes;
    wrows_tile_mma_n<NC, TPW, TPW>(nt, acc, p, slot0, sx, sy, dhi, any);
    wgmma_wait<0>();
#pragma unroll
    for (int t = 0; t < TPW; ++t) fence_regs(acc[t]);
    any = true;
    if (lane == 0) mbar_arrive(&empty_bar[st]);
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

// launches the partial-sum kernel; *slices_out = number of partial slices written to ws (each slice_elems floats:
// dW3 [Cout,3,3,Cin] then, with dy1, dW1 [Cout,Cin]). Returns 0 / -1 (not eligible) / -2 (launch failure).
int hb_wgrad_rows_try(const void* x, const void* dy, const void* dy1, float* ws, size_t ws_bytes, int N, int H, int W, int Cin,
                      int Cout, int num_ctas, cudaStream_t stream, int* slices_out) {
  WRowsPlan pl{};
  const int has_b1 = dy1 != nullptr;
  if (!plan_wrows(pl, N, H, W, Cin, Cout, num_ctas, has_b1)) return -1;
  WRowsParams& p = pl.p;
  if (!ws || ws_bytes < (size_t)pl.members * p.slice_elems * sizeof(float)) return -1;
  p.ws = ws;
  CUtensorMap tmX, tmDY, tmDY1;
  {
    uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)N};
    uint64_t strides[3] = {(uint64_t)Cin * 2, (uint64_t)W * Cin * 2, (uint64_t)H * W * Cin * 2};
    uint32_t box[4] = {64, (uint32_t)p.Wp, (uint32_t)(p.TRO + 2), 1};
    if (tmap::encode_tiled_bf16(&tmX, x, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B)) return -1;
    uint64_t ydims[4] = {(uint64_t)Cout, (uint64_t)W, (uint64_t)H, (uint64_t)N};
    uint64_t ystrides[3] = {(uint64_t)Cout * 2, (uint64_t)W * Cout * 2, (uint64_t)H * W * Cout * 2};
    uint32_t ybox[4] = {64, (uint32_t)p.Wp, (uint32_t)p.TRO, 1};
    if (tmap::encode_tiled_bf16(&tmDY, dy, 4, ydims, ystrides, ybox, CU_TENSOR_MAP_SWIZZLE_128B)) return -1;
    if (tmap::encode_tiled_bf16(&tmDY1, has_b1 ? dy1 : dy, 4, ydims, ystrides, ybox, CU_TENSOR_MAP_SWIZZLE_128B)) return -1;
  }
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(conv_wgrad_rows_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess ||
        cudaFuncSetAttribute(conv_wgrad_rows_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess ||
        cudaFuncSetAttribute(conv_wgrad_rows_kernel<48>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess ||
        cudaFuncSetAttribute(conv_wgrad_rows_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess)
      return -1;
    attr_set = true;
  }
  if (pl.smem > 227 * 1024) return -1;
  switch (p.co_group) {
    case 16: conv_wgrad_rows_kernel<16><<<pl.grid, kThreads, pl.smem, stream>>>(tmX, tmDY, tmDY1, p); break;
    case 32: conv_wgrad_rows_kernel<32><<<pl.grid, kThreads, pl.smem, stream>>>(tmX, tmDY, tmDY1, p); break;
    case 48: conv_wgrad_rows_kernel<48><<<pl.grid, kThreads, pl.smem, stream>>>(tmX, tmDY, tmDY1, p); break;
    default: conv_wgrad_rows_kernel<64><<<pl.grid, kThreads, pl.smem, stream>>>(tmX, tmDY, tmDY1, p); break;
  }
  g_hb_launches.fetch_add(1, std::memory_order_relaxed);
  *slices_out = pl.members;
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}
