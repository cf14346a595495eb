// "Row-window" 3x3 convolution (stride 1, pad 1) for the HBM/L2-bound layers (Cin <= 128, all filter taps resident
// in shared memory): the input rows needed by a band of output rows are brought in ONCE per tile by a single tiled TMA
// load (with a one-pixel zero halo supplied by TMA's out-of-bounds fill) and all nine filter taps are issued as
// *shifted windows of that one buffer* - a wgmma shared-memory descriptor may start at any 128-byte row of a
// 128B-swizzled TMA buffer because the swizzle is a function of the absolute shared-memory address.
//
// Why: the generic implicit-GEMM kernel (conv_fprop.cu) issues one im2col TMA load per tap, i.e. it reads every input
// element 9x from L2. Here a tile of TRO output rows loads TRO+2 input rows: 1.3-2x instead of 9x.
//
// Geometry. Shared-memory row pitch Wp = W + 2 pixels (128 B each = one 64-channel block). A "sub-tile" is one
// M = 128 tile (two 64-row warpgroup MMAs) covering SR = floor(128 / Wp) output rows laid out with the SAME pitch Wp
// (so 2 junk columns per row); for tap (r, s) its A operand is the buffer window starting at pixel row
// (sub*SR + r) * Wp + s. Junk accumulator rows (q >= W, rows past the image) are skipped by the epilogue. The filter
// (all 9 taps x channel blocks) is loaded once per CTA and stays resident.
//
// Warp roles: one TMA producer warpgroup and two consumer warpgroups (rows 0-63 and 64-127 of every sub-tile) that
// issue the wgmma chain of a sub-tile and then run its epilogue (accumulator registers -> bf16 staging tile in shared
// memory -> coalesced 128-bit stores); the producer meanwhile loads the next tile's rows into the other ring slot.
#include "conv_common.cuh"

namespace {

using namespace tc;
using namespace conv;

struct RowsParams {
  int N, H, W, Cin, Cout;
  int Wp;        // smem row pitch in pixels (W + 2)
  int SR;        // output rows per sub-tile (one M=128 tile)
  int NSUB;      // sub-tiles per tile
  int TRO;       // output rows per tile = SR * NSUB
  int CB;        // 64-channel blocks
  int ksteps_last;  // k-steps (of 16 channels) in the last channel block
  int tiles_per_img, num_tiles;
  int nstages;       // ring slots: 2, or 1 when two tiles' rows do not fit in shared memory
  int stage_bytes;   // CB * (cb_bytes + nextra * ecb_bytes): the main rows and every extra source of one tile
  int cb_bytes;      // bytes of one 64-channel block buffer of the main rows, rounded to 1024
  int ecb_bytes;     // same for an extra source (no halo rows)
  int w_tap_bytes;   // BN * 128 rounded to 1024
  int out_pitch;
  int act;
  int nextra;        // 0..2 additional "centre tap only" sources accumulated into the same output (see below)
  __nv_bfloat16* y;
  const float* bias;
  const __nv_bfloat16* residual;
  float* stats;      // optional statistics of the bf16 output, 2 * gridDim.x slots (conv_common.cuh)
};

// BN = Cout (a multiple of 16 up to 128), the N of every wgmma
template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
conv_rows_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW,
                 const __grid_constant__ CUtensorMap tmXe0, const __grid_constant__ CUtensorMap tmWe0,
                 const __grid_constant__ CUtensorMap tmXe1, const __grid_constant__ CUtensorMap tmWe1, const RowsParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* wsm = smem;                                          // [9 + nextra][CB][BN x 128 B]
  uint8_t* stage0 = wsm + (size_t)(9 + p.nextra) * p.CB * p.w_tap_bytes;     // ring of nstages tile buffers
  uint8_t* sout = stage0 + (size_t)p.nstages * p.stage_bytes;   // [128][out_pitch]
  const size_t sout_bytes = ((size_t)128 * p.out_pitch + 15) & ~size_t(15);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sout + sout_bytes);
  uint64_t* full_bar = bars;        // [2]
  uint64_t* empty_bar = bars + 2;   // [2]
  uint64_t* w_bar = bars + 4;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmX);
    prefetch_tmap(&tmW);
    for (int i = 0; i < 2; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kConsumers / 32); }
    mbar_init(w_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ================= TMA producer =================
    if (warp == 0 && lane == 0) {
      prefetch_tmap(&tmXe0); prefetch_tmap(&tmWe0); prefetch_tmap(&tmXe1); prefetch_tmap(&tmWe1);
      // resident filters: 9 taps x CB channel blocks (+ one 1x1 filter per extra source)
      mbar_arrive_expect_tx(w_bar, (uint32_t)((9 + p.nextra) * p.CB * BN * 128));
      for (int tap = 0; tap < 9; ++tap)
        for (int cb = 0; cb < p.CB; ++cb)
          tma_load_3d(&tmW, w_bar, wsm + (size_t)(tap * p.CB + cb) * p.w_tap_bytes, cb * 64, tap, 0);
      for (int e = 0; e < p.nextra; ++e)
        for (int cb = 0; cb < p.CB; ++cb)
          tma_load_3d(e == 0 ? &tmWe0 : &tmWe1, w_bar, wsm + (size_t)((9 + e) * p.CB + cb) * p.w_tap_bytes, cb * 64, 0, 0);
      const uint32_t tx = (uint32_t)(p.CB * ((p.TRO + 2) + p.nextra * p.TRO) * p.Wp * 128);
      int it = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++it) {
        const int n = tile / p.tiles_per_img, p0 = (tile % p.tiles_per_img) * p.TRO;
        const Ring ring = Ring::at(it, p.nstages);
        mbar_wait(&empty_bar[ring.stage], ring.phase ^ 1);
        mbar_arrive_expect_tx(&full_bar[ring.stage], tx);
        for (int b = 0; b <= p.nextra; ++b) {
          const CUtensorMap* tm = b == 0 ? &tmX : (b == 1 ? &tmXe0 : &tmXe1);
          const int h0 = b == 0 ? p0 - 1 : p0;   // the extra sources need no row halo (centre tap only)
          for (int cb = 0; cb < p.CB; ++cb) {
            // box (64 ch, Wp, rows, 1 image) at (c, w = -1, h0, n): halo and image borders = OOB zero fill
            tma_load_4d(tm, &full_bar[ring.stage],
                        stage0 + (size_t)ring.stage * p.stage_bytes +
                            (size_t)p.CB * (b ? p.cb_bytes + (b - 1) * p.ecb_bytes : 0) +
                            (size_t)cb * (b ? p.ecb_bytes : p.cb_bytes),
                        cb * 64, -1, h0, n);
          }
        }
      }
    }
    return;
  }

  // ================= consumers =================
  const int et = threadIdx.x - 128;          // 0..255
  const int wg = et >> 7;                    // rows [64*wg, 64*wg + 64) of every sub-tile
  const int frow = 64 * wg + frag_row(et & 127);
  const int fcol = frag_col(et & 127);
  const uint32_t dhi = desc_hi(1024);
  const uint32_t w_lo0 = desc_lo(smem_u32(wsm), 16);
  const uint32_t w_tap_lo = (uint32_t)p.w_tap_bytes >> 4;
  const uint32_t cb_lo = (uint32_t)p.cb_bytes >> 4;
  const uint32_t ecb_lo = (uint32_t)p.ecb_bytes >> 4;
  const int chunks_per_row = BN / 8;
  // column statistics: thread = (column pair pr, pixel subset rg) over the valid pixels of every sub-tile
  const int npairs = BN >> 1, rgs = kConsumers / npairs;
  const int st_rg = et / npairs, st_pr = et - st_rg * npairs;
  const bool st_on = p.stats != nullptr && st_rg < rgs;
  float4 stat = make_float4(0.f, 0.f, 0.f, 0.f);
  float acc[64];
  mbar_wait(w_bar, 0);
  int it = 0;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++it) {
    const int n = tile / p.tiles_per_img, p0 = (tile % p.tiles_per_img) * p.TRO;
    const Ring ring = Ring::at(it, p.nstages);
    mbar_wait(&full_bar[ring.stage], ring.phase);
    // window start of this warpgroup's 64 rows: 64 pixel rows x 128 B further
    const uint32_t s_lo =
        desc_lo(smem_u32(stage0 + (size_t)ring.stage * p.stage_bytes), 16) + (uint32_t)wg * ((64 * 128) >> 4);
    for (int sub = 0; sub < p.NSUB; ++sub) {
      // one commit group per (tap or extra source, channel block), all in flight until the sub-tile's epilogue
#pragma unroll 1
      for (int tap = 0; tap < 9; ++tap) {
        const int r = tap / 3, s = tap % 3;
        // 128-byte pixel rows: (row index) * 128 B >> 4 = row index * 8
        uint32_t a_lo = s_lo + (uint32_t)(((sub * p.SR + r) * p.Wp + s) * 8);
        uint32_t b_lo = w_lo0 + (uint32_t)(tap * p.CB) * w_tap_lo;
        for (int cb = 0; cb < p.CB; ++cb) {
          const int ks = (cb == p.CB - 1) ? p.ksteps_last : 4;
          wgmma_group_ks<BN, 0, 0>(ks, acc, a_lo, b_lo, 2, dhi, (tap | cb) ? 1u : 0u);
          a_lo += cb_lo;
          b_lo += w_tap_lo;
        }
      }
      for (int e = 0; e < p.nextra; ++e) {
        // centre-tap source: buffer row 0 is output row p0, columns start at w = -1 -> window offset 1 pixel
        uint32_t a_lo = s_lo + (uint32_t)p.CB * (cb_lo + e * ecb_lo) + (uint32_t)((sub * p.SR * p.Wp + 1) * 8);
        uint32_t b_lo = w_lo0 + (uint32_t)((9 + e) * p.CB) * w_tap_lo;
        for (int cb = 0; cb < p.CB; ++cb) {
          const int ks = (cb == p.CB - 1) ? p.ksteps_last : 4;
          wgmma_group_ks<BN, 0, 0>(ks, acc, a_lo, b_lo, 2, dhi, 1u);
          a_lo += ecb_lo;
          b_lo += w_tap_lo;
        }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (sub == p.NSUB - 1 && lane == 0) mbar_arrive(&empty_bar[ring.stage]);   // ring slot may be refilled

      // ---- epilogue of this sub-tile ----
      consumer_sync();   // staging tile free
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = 8 * j + fcol;
        if (col < BN) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
            if (p.bias) { f0 += __ldg(p.bias + col); f1 += __ldg(p.bias + col + 1); }
            if (p.act == 1 && !p.residual) { f0 = hb::relu_nan(f0); f1 = hb::relu_nan(f1); }
            *reinterpret_cast<__nv_bfloat162*>(sout + (size_t)(frow + 8 * h) * p.out_pitch + col * 2) =
                __floats2bfloat162_rn(f0, f1);
          }
        }
      }
      consumer_sync();   // staged tile visible
      // copy-out: iterate over the VALID output pixels of this sub-tile (row-major), 16-byte chunks
      const int row0 = p0 + sub * p.SR;
      const int rows_valid = max(0, min(p.SR, min(p.H, p0 + p.TRO) - row0));
      const int total = rows_valid * p.W * chunks_per_row;
      // division-free walk: thread `et` starts at chunk et of the valid pixels and advances by 256 chunks per trip
      int pix0 = et / chunks_per_row;
      int c8 = et - pix0 * chunks_per_row;
      int i = pix0 / p.W, q = pix0 - i * p.W;
      const int dpix = kConsumers / chunks_per_row, dc = kConsumers - dpix * chunks_per_row;
      const int di = dpix / p.W, dq = dpix - di * p.W;
      for (int ch = et; ch < total; ch += kConsumers) {
        uint4 val = *reinterpret_cast<const uint4*>(sout + (size_t)(i * p.Wp + q) * p.out_pitch + c8 * 16);
        const size_t off = ((size_t)(n * p.H + row0 + i) * p.W + q) * p.Cout + c8 * 8;
        if (p.residual) {
          const uint4 rv = *reinterpret_cast<const uint4*>(p.residual + off);
          add_residual16(val, rv, p.act == 1);
        }
        *reinterpret_cast<uint4*>(p.y + off) = val;
        c8 += dc; q += dq; i += di;
        if (c8 >= chunks_per_row) { c8 -= chunks_per_row; ++q; }
        if (q >= p.W) { q -= p.W; ++i; }
      }
      if (st_on && !p.residual) {
        // statistics of the staged bf16 tile over its valid pixels (junk columns q >= W and rows past the image skipped)
        const int npix = rows_valid * p.W;
        int si = st_rg / p.W, sq = st_rg - si * p.W;
        const int sdi = rgs / p.W, sdq = rgs - sdi * p.W;
        const uint8_t* sp = sout + st_pr * 4;
        for (int v = st_rg; v < npix; v += rgs) {
          accum_pair(stat, sp + (size_t)(si * p.Wp + sq) * p.out_pitch);
          sq += sdq; si += sdi;
          if (sq >= p.W) { sq -= p.W; ++si; }
        }
      }
    }
  }
  if (p.stats) {
    // fold the pixel subsets in a fixed order into slot 2*blockIdx.x; slot 2*blockIdx.x + 1 is written as zeros (every
    // (slot, channel) is written)
    consumer_sync();
    float4* scratch = reinterpret_cast<float4*>(sout);   // [256] float4, 4 KB <= staging tile
    scratch[et] = stat;
    consumer_sync();
    if (et < 2 * BN) {
      const int c = et % BN, half = et / BN;
      store_stats(p.stats, blockIdx.x * 2 + half, p.Cout, c,
                  half == 0 ? fold_stats(scratch, rgs, npairs, c) : make_float2(0.f, 0.f));
    }
  }
}

}  // namespace

// Called from hb_conv2d_fused_bf16 and hb_conv3x3_accum_bf16 (declared in conv_common.cuh).
int hb_conv_rows_try(const void* x, const void* w, void* y, const float* bias, const void* residual, int N, int H, int W,
                     int Cin, int Cout, int act, int num_ctas, cudaStream_t stream, int nextra, const void* const* xe,
                     const void* const* we, float* stats, int* stat_slots) {
  constexpr int kNo = (int)cudaErrorNotSupported;
  if (stats && (residual || !stat_slots)) return kNo;
  if (Cout % 16 != 0 || Cout > 128 || Cin % 8 != 0 || Cin > 128) return kNo;
  const int Wp = W + 2;
  if (Wp > 128 || W < 8 || nextra < 0 || nextra > 2) return kNo;
  RowsParams p{};
  p.N = N; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.Wp = Wp; p.nextra = nextra;
  p.SR = 128 / Wp;
  p.CB = (Cin + 63) / 64;
  const int last = Cin - (p.CB - 1) * 64;
  p.ksteps_last = (last + 15) / 16;
  p.w_tap_bytes = ((Cout * 128) + 1023) & ~1023;
  p.out_pitch = Cout * 2 + 16;
  const int w_bytes = (9 + nextra) * p.CB * p.w_tap_bytes;
  const int out_bytes = (((128 * p.out_pitch + 15) & ~15) + 1023) & ~1023;   // one staging tile
  const int budget = 222 * 1024 - w_bytes - out_bytes - 256;
  // largest NSUB whose ring buffers (main rows + every extra source) fit in shared memory: two ring slots if
  // possible, else one (the next tile's rows then load while the epilogue of the last sub-tile runs)
  const int max_rows_needed = (H + p.SR - 1) / p.SR;
  int nsub = 0;
  for (int nst = 2; nst >= 1 && nsub < 1; --nst) {
    for (nsub = max_rows_needed < 8 ? max_rows_needed : 8; nsub >= 1; --nsub) {
      const int tro = nsub * p.SR;
      // the last sub-tile's windows read up to 127 + 2*Wp + 2 pixel rows past its first row: keep them inside the buffer
      const int reach = (((nsub - 1) * p.SR + 2) * Wp + 2 + 128) * 128;
      const int rows = (tro + 2) * Wp * 128;
      const int need = ((rows > reach ? rows : reach) + 1023) & ~1023;
      const int ereach = ((nsub - 1) * p.SR * Wp + 1 + 128) * 128, erows = tro * Wp * 128;
      const int eneed = ((erows > ereach ? erows : ereach) + 1023) & ~1023;
      if (nst * p.CB * (need + nextra * eneed) <= budget) {
        p.nstages = nst; p.cb_bytes = need; p.ecb_bytes = eneed;
        break;
      }
    }
  }
  if (nsub < 1) return kNo;
  p.NSUB = nsub;
  p.TRO = nsub * p.SR;
  p.stage_bytes = p.CB * (p.cb_bytes + nextra * p.ecb_bytes);
  p.tiles_per_img = (H + p.TRO - 1) / p.TRO;
  p.num_tiles = N * p.tiles_per_img;
  p.act = act;
  p.y = (__nv_bfloat16*)y; p.bias = bias; p.residual = (const __nv_bfloat16*)residual;
  p.stats = stats;

  CUtensorMap tmX, tmW, tmXe[2], tmWe[2];
  if (tmap::encode_nhwc_box(&tmX, x, N, H, W, Cin, Wp, p.TRO + 2)) return kNo;
  if (tmap::encode_krsc_slab(&tmW, w, Cout, 9, Cin, Cout)) return kNo;
  for (int e = 0; e < 2; ++e) {
    // unused slots alias the main tensors (never dereferenced by the kernel)
    const void* xs = e < nextra ? xe[e] : x;
    const void* ws = e < nextra ? we[e] : w;
    if (!hb::aligned16(xs) || !hb::aligned16(ws)) return kNo;
    if (tmap::encode_nhwc_box(&tmXe[e], xs, N, H, W, Cin, Wp, p.TRO)) return kNo;
    if (tmap::encode_krsc_slab(&tmWe[e], ws, Cout, 1, Cin, Cout)) return kNo;
  }
  const size_t smem_bytes = (size_t)w_bytes + (size_t)p.nstages * p.stage_bytes + out_bytes + 64 + 1024;
  if (smem_bytes > 227 * 1024) return kNo;
  int grid = num_ctas > 0 ? num_ctas : HB_NUM_SMS;
  if (grid > p.num_tiles) grid = p.num_tiles;
  if (stat_slots) *stat_slots = 2 * grid;
  // one instantiation per Cout
  return (int)dispatch_width<16, 128>(Cout, [&](auto bn) {
    return launch<conv_rows_kernel<decltype(bn)::value>>(grid, smem_bytes, stream, tmX, tmW, tmXe[0], tmWe[0], tmXe[1],
                                                          tmWe[1], p);
  });
}

extern "C" {

// y[N,H,W,Cout] = conv3x3(x, w; stride 1, pad 1) + sum_{e < nextra} conv1x1(xe[e], we[e])    (all NHWC bf16, Cin channels)
// One kernel, one accumulator: used for the input gradient of a RepVGG block,
//   dX = dgrad3x3(dY3) + dgrad1x1(dY1) + I * dX_identity
// (reference: the three autograd contributions of models/classification/repvgg.py:71-73 summed by two add kernels).
// Returns cudaErrorNotSupported (801) without launching when the shape does not fit the shared-memory-resident scheme;
// callers then fall back to separate convolutions. Otherwise 0, or the launch's error.
int hb_conv3x3_accum_bf16(const void* x, const void* w, const void* xe0, const void* we0, const void* xe1, const void* we1,
                          int nextra, void* y, int N, int H, int W, int Cin, int Cout, int num_ctas, void* stream) {
  const void* xe[2] = {xe0, xe1};
  const void* we[2] = {we0, we1};
  if (!hb::aligned16(x) || !hb::aligned16(w) || !hb::aligned16(y)) return (int)cudaErrorMisalignedAddress;
  return hb_conv_rows_try(x, w, y, nullptr, nullptr, N, H, W, Cin, Cout, 0, num_ctas, (cudaStream_t)stream, nextra, xe, we,
                          nullptr, nullptr);
}

}  // extern "C"
