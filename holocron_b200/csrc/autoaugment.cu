// Batched TrivialAugmentWide (torchvision.transforms.TrivialAugmentWide.forward and the autoaugment _apply_op it calls,
// the third random transform of the reference's classification recipe, references/classification/train.py:103), on
// uint8 images of one shape: at most two launches per batch, whatever its op mix, and no host synchronisation.
//
// Image n is one row of a device table (AugDesc, uploaded by the caller from pinned memory together with the fp32
// parameters and the list of images that need statistics): a strided source [C][H][W] read in place, a contiguous
// destination [C][H][W], the op drawn for it and that op's parameters. The arithmetic is torchvision's tensor path on
// CUDA (_functional_tensor.py), fp32 operation by fp32 operation, with no contraction into FMAs where torch runs the
// products and the sum as separate kernels:
//   blend (Brightness b = 0, Contrast b = grayscale mean, Color b = pixel grayscale, Sharpness b = blurred pixel):
//       trunc(clamp(f32(r)*v + f32(1 - r)*b, 0, 255))
//   grayscale: trunc((0.2989*r + 0.587*g) + 0.114*b)
//   Posterize v & mask; Solarize v >= f32(t) ? 255 - v : v;
//   AutoContrast trunc(clamp((v - min) * (1 / (max - min) * 255)))
//   Equalize: histc, step = floor(sum of the nonzero bins but the last / 255), lut = floor((cumsum + step/2) / step)
//   ShearX/Y, TranslateX/Y, Rotate: _gen_affine_grid and grid_sample(align_corners=False, zeros) with the optional
//       fill mask, torch.round to uint8.
//
// Launch 1 (only when an image drew Contrast, AutoContrast or Equalize): one CTA per (image, channel, pixel slice)
// counts a 256-bin int32 histogram in shared memory and writes it to scratch[row][slice][256], row = 3*k + channel for
// the k-th image with statistics (Contrast of an RGB image: row 3*k holds its uint8 grayscale). Integer counts are
// order-free, so two runs give the same bits; no global atomics and no memset.
// Launch 2: one CTA per (image, tile of output rows); the op is CTA-uniform. A thread owns a 16-pixel chunk of one
// output row for every channel. Per-channel value maps build a 256-entry LUT per channel in shared memory (from the
// histogram slices, summed in slice order, where the op needs statistics) and apply it with 16-byte loads and stores
// where rows are contiguous and aligned; Color reads the three channels of a pixel; Sharpness reads its 3x3 stencil
// through L1; the affine ops gather 1 or 4 taps per channel from fp32 coordinates computed once per pixel.
#include "pixel.cuh"

using namespace hb;

namespace {

constexpr int kThreads = 256;

// op codes: the order of TrivialAugmentWide._augmentation_space
enum Op {
  kIdentity = 0, kShearX, kShearY, kTranslateX, kTranslateY, kRotate, kBrightness, kColor, kContrast, kSharpness,
  kPosterize, kSolarize, kAutoContrast, kEqualize
};
// fp32 parameters of one image (16 floats): ratio r, 1 - r, solarize threshold, the inverse affine matrix, the fill
enum Param { kR = 0, kQ = 1, kThreshold = 2, kMatrix = 3, kFill = 9 };

// One row of the descriptor table (16 x int64, include/holocron_b200.h). Pointers are addresses, strides count elements
// (bytes).
struct AugDesc {
  long long src, dst, sc, sh, sw, C, H, W, op, stat, mask, fill, bilinear, reserved0, reserved1, reserved2;
};

__device__ __forceinline__ bool needs_stats(int op) {
  return op == kContrast || op == kAutoContrast || op == kEqualize;
}

__global__ void __launch_bounds__(kThreads) histogram_kernel(const AugDesc* __restrict__ descs,
                                                             const long long* __restrict__ stat_images,
                                                             int* __restrict__ scratch, int slices) {
  __shared__ int hist[256];
  const int s = blockIdx.x % slices, row = blockIdx.x / slices;
  const int k = row / 3, c = row - 3 * k;
  const AugDesc& d = descs[stat_images[k]];
  const int C = (int)d.C;
  const bool to_gray = d.op == kContrast && C == 3;
  if (to_gray ? c > 0 : c >= C) return;
  hist[threadIdx.x] = 0;
  __syncthreads();
  const Slice sl = pixel_slice(d, s, slices);
  for (long long p = sl.p0 + threadIdx.x; p < sl.p1; p += kThreads) {
    const uint8_t* px = pixel_at<uint8_t>(d, p);
    const uint8_t v = to_gray ? gray(px[0], px[d.sc], px[2 * d.sc]) : px[c * d.sc];
    atomicAdd(&hist[v], 1);
  }
  __syncthreads();
  scratch[((long long)row * slices + s) * 256 + threadIdx.x] = hist[threadIdx.x];
}

// The per-channel LUTs of a value-map op, built by the whole CTA (thread t computes entry t of every channel).
__device__ void build_luts(const AugDesc& d, const float* P, const int* __restrict__ scratch, int slices,
                           uint8_t (*lut)[256], int (*cnt)[256]) {
  const int t = threadIdx.x, op = (int)d.op, C = (int)d.C;
  const float r = P[kR], q = P[kQ];
  const int rows = op == kContrast ? 1 : C;
  if (needs_stats(op)) {
    for (int c = 0; c < rows; ++c) {
      const int* h = scratch + (3 * d.stat + c) * slices * 256LL + t;
      int sum = 0;
      for (int s = 0; s < slices; ++s) sum += h[s * 256];
      cnt[c][t] = sum;
    }
  }
  __syncthreads();
  if (op == kContrast) {
    const long long sum = ordered_block_sum<kThreads>((long long)t * cnt[0][t]);
    // torch's CUDA mean: the fp32 sum times the fp32 factor 1 / numel
    const float mean = __fmul_rn((float)sum, __fdiv_rn(1.f, (float)(d.H * d.W)));
    const uint8_t out = blend(r, q, (uint8_t)t, mean);
    for (int c = 0; c < C; ++c) lut[c][t] = out;
    return;
  }
  if (op == kAutoContrast) {
    __shared__ int lo[3], hi[3];
    if (t < 3) lo[t] = 255, hi[t] = 0;
    __syncthreads();
    for (int c = 0; c < C; ++c)
      if (cnt[c][t] != 0) atomicMin(&lo[c], t), atomicMax(&hi[c], t);
    __syncthreads();
    for (int c = 0; c < C; ++c) {
      float mn = (float)lo[c];
      // torch's 255 / t is t.reciprocal() * 255: two roundings
      float scale = __fmul_rn(__frcp_rn(__fsub_rn((float)hi[c], mn)), 255.f);
      if (!isfinite(scale)) mn = 0.f, scale = 1.f;
      lut[c][t] = trunc_u8(__fmul_rn(__fsub_rn((float)t, mn), scale));
    }
    return;
  }
  if (op == kEqualize) {
    __shared__ int step[3];
    // warp c scans channel c: inclusive cumulative counts in place, then the step from the total and the last bin
    const int w = t >> 5, lane = t & 31;
    if (w < C) {
      int* h = cnt[w];
      int run = 0, last = 0;
      int local[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int v = h[lane * 8 + i];
        if (v != 0) last = v;
        run += v;
        local[i] = run;
      }
      int incl = run;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += u;
      }
      const int total = __shfl_sync(0xffffffffu, incl, 31);
      // count of the last nonzero bin: from the highest lane holding one
      const unsigned has = __ballot_sync(0xffffffffu, last != 0);
      const int top_last = __shfl_sync(0xffffffffu, last, 31 - __clz(has));
      __syncwarp();
#pragma unroll
      for (int i = 0; i < 8; ++i) h[lane * 8 + i] = incl - run + local[i];
      if (lane == 0) step[w] = (total - top_last) / 255;
    }
    __syncthreads();
    for (int c = 0; c < C; ++c) {
      const int st = step[c];
      lut[c][t] = st == 0 ? (uint8_t)t : t == 0 ? 0 : (uint8_t)min(255, (cnt[c][t - 1] + st / 2) / st);
    }
    return;
  }
  uint8_t out = (uint8_t)t;
  if (op == kBrightness) out = blend(r, q, (uint8_t)t, 0.f);
  else if (op == kPosterize) out = (uint8_t)(t & (int)d.mask);
  else if (op == kSolarize) out = (float)t >= P[kThreshold] ? (uint8_t)(255 - t) : (uint8_t)t;
  for (int c = 0; c < C; ++c) lut[c][t] = out;
}

__global__ void __launch_bounds__(kThreads) apply_kernel(const AugDesc* __restrict__ descs,
                                                         const float* __restrict__ params,
                                                         const int* __restrict__ scratch, int slices,
                                                         int rows_per_tile, int tiles) {
  __shared__ uint8_t lut[3][256];
  __shared__ int cnt[3][256];
  const int n = blockIdx.x / tiles;
  const AugDesc& d = descs[n];
  const float* P = params + 16LL * n;
  const int C = (int)d.C, H = (int)d.H, W = (int)d.W;
  int op = (int)d.op;
  // torchvision returns these images unchanged
  if ((op == kColor && C == 1) || (op == kSharpness && (H <= 2 || W <= 2))) op = kIdentity;
  const bool is_lut = op == kIdentity || op == kBrightness || op == kContrast || op == kPosterize ||
                      op == kSolarize || op == kAutoContrast || op == kEqualize;
  if (is_lut) {
    build_luts(d, P, scratch, slices, lut, cnt);
    __syncthreads();
  }
  const uint8_t* src = reinterpret_cast<const uint8_t*>(d.src);
  uint8_t* dst = reinterpret_cast<uint8_t*>(d.dst);
  const long long sc = d.sc, sh = d.sh, sw = d.sw;
  const float r = P[kR], q = P[kQ];
  const RowTile tile(n, tiles, rows_per_tile, H, W);
  // geometric ops: theta^T / [w/2, h/2] as _gen_affine_grid forms it
  const float hw = 0.5f * (float)W, hh = 0.5f * (float)H;
  const float ax = __fdiv_rn(P[kMatrix], hw), bx = __fdiv_rn(P[kMatrix + 1], hw), cx = __fdiv_rn(P[kMatrix + 2], hw);
  const float ay = __fdiv_rn(P[kMatrix + 3], hh), by = __fdiv_rn(P[kMatrix + 4], hh),
              cy = __fdiv_rn(P[kMatrix + 5], hh);
  const bool has_fill = d.fill != 0, bilinear = d.bilinear != 0;

  for (int item = threadIdx.x; item < tile.items(); item += kThreads) {
    const auto [y, x0, len] = Chunk(tile, item, W);
    const uint8_t* srow = src + y * sh + x0 * sw;
    uint8_t* drow = dst + ((long long)y * W + x0);
    const long long plane = (long long)H * W;
    if (is_lut) {
      for (int c = 0; c < C; ++c) {
        Vec16<uint8_t> v = load_chunk(srow + c * sc, sw, len);
#pragma unroll
        for (int j = 0; j < kChunk; ++j) v.v[j] = lut[c][v.v[j]];
        store_chunk(drow + c * plane, v, len);
      }
    } else if (op == kColor) {
      Vec16<uint8_t> vr = load_chunk(srow, sw, len), vg = load_chunk(srow + sc, sw, len),
                     vb = load_chunk(srow + 2 * sc, sw, len);
#pragma unroll
      for (int j = 0; j < kChunk; ++j) {
        const float g = (float)gray(vr.v[j], vg.v[j], vb.v[j]);
        vr.v[j] = blend(r, q, vr.v[j], g);
        vg.v[j] = blend(r, q, vg.v[j], g);
        vb.v[j] = blend(r, q, vb.v[j], g);
      }
      store_chunk(drow, vr, len);
      store_chunk(drow + plane, vg, len);
      store_chunk(drow + 2 * plane, vb, len);
    } else if (op == kSharpness) {
      const bool edge_row = y == 0 || y == H - 1;
      for (int c = 0; c < C; ++c) {
        const uint8_t* p = srow + c * sc;
        Vec16<uint8_t> o;
#pragma unroll
        for (int j = 0; j < kChunk; ++j) {
          if (j >= len) continue;
          const uint8_t* pj = p + j * sw;
          const int v = __ldg(pj);
          int blurred = v;  // the one-pixel border keeps its value, and still goes through the blend
          if (!edge_row && x0 + j > 0 && x0 + j < W - 1) {
            // [1 1 1; 1 5 1; 1 1 1] / 13, rounded: the exact sum is an integer over 13, never a rounding tie
            int s = 4 * v;
#pragma unroll
            for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
              for (int dx = -1; dx <= 1; ++dx) s += __ldg(pj + dy * sh + dx * sw);
            blurred = (2 * s + 13) / 26;
          }
          o.v[j] = blend(r, q, (uint8_t)v, (float)blurred);
        }
        store_chunk(drow + c * plane, o, len);
      }
    } else {
      Vec16<uint8_t> o[3];
      const float yb = (float)(2 * y - H + 1) * 0.5f;
#pragma unroll
      for (int j = 0; j < kChunk; ++j) {
        if (j >= len) continue;
        const float xb = (float)(2 * (x0 + j) - W + 1) * 0.5f;
        const float gx = __fadd_rn(__fmaf_rn(yb, bx, __fmul_rn(xb, ax)), cx);
        const float gy = __fadd_rn(__fmaf_rn(yb, by, __fmul_rn(xb, ay)), cy);
        // grid_sample's unnormalisation with align_corners=False
        const float ix = __fmaf_rn(__fadd_rn(gx, 1.f), (float)W, -1.f) * 0.5f;
        const float iy = __fmaf_rn(__fadd_rn(gy, 1.f), (float)H, -1.f) * 0.5f;
        if (!bilinear) {
          const int xi = __float2int_rn(ix), yi = __float2int_rn(iy);
          const bool in = xi >= 0 && xi < W && yi >= 0 && yi < H;
          const uint8_t* pj = src + (long long)yi * sh + (long long)xi * sw;
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            if (c >= C) break;
            o[c].v[j] = in ? pj[c * sc] : has_fill ? (uint8_t)__float2int_rn(P[kFill + c]) : 0;
          }
        } else {
          const int xw = __float2int_rd(ix), yn = __float2int_rd(iy);
          const float fxw = (float)xw, fxe = (float)(xw + 1), fyn = (float)yn, fys = (float)(yn + 1);
          const float nw = __fmul_rn(__fsub_rn(fxe, ix), __fsub_rn(fys, iy));
          const float ne = __fmul_rn(__fsub_rn(ix, fxw), __fsub_rn(fys, iy));
          const float sw_ = __fmul_rn(__fsub_rn(fxe, ix), __fsub_rn(iy, fyn));
          const float se = __fmul_rn(__fsub_rn(ix, fxw), __fsub_rn(iy, fyn));
          const bool xw_in = xw >= 0 && xw < W, xe_in = xw + 1 >= 0 && xw + 1 < W;
          const bool yn_in = yn >= 0 && yn < H, ys_in = yn + 1 >= 0 && yn + 1 < H;
          const uint8_t* pnw = src + (long long)yn * sh + (long long)xw * sw;
          float m = 0.f;
          if (yn_in && xw_in) m = __fadd_rn(m, nw);
          if (yn_in && xe_in) m = __fadd_rn(m, ne);
          if (ys_in && xw_in) m = __fadd_rn(m, sw_);
          if (ys_in && xe_in) m = __fadd_rn(m, se);
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            if (c >= C) break;
            const uint8_t* pc = pnw + c * sc;
            float acc = 0.f;
            if (yn_in && xw_in) acc = __fmaf_rn((float)pc[0], nw, acc);
            if (yn_in && xe_in) acc = __fmaf_rn((float)pc[sw], ne, acc);
            if (ys_in && xw_in) acc = __fmaf_rn((float)pc[sh], sw_, acc);
            if (ys_in && xe_in) acc = __fmaf_rn((float)pc[sh + sw], se, acc);
            if (has_fill) acc = __fadd_rn(__fmul_rn(acc, m), __fmul_rn(__fsub_rn(1.f, m), P[kFill + c]));
            o[c].v[j] = (uint8_t)__float2int_rn(acc);
          }
        }
      }
#pragma unroll
      for (int c = 0; c < 3; ++c)
        if (c < C) store_chunk(drow + c * plane, o[c], len);
    }
  }
}

}  // namespace

extern "C" int hb_autoaugment_batch(const void* descs, const float* params, const long long* stat_images, int* scratch,
                                    int N, int n_stat, int H, int W, int slices, void* stream) {
  if (N <= 0 || n_stat < 0 || n_stat > N || H <= 0 || W <= 0 || slices <= 0) return (int)cudaErrorInvalidValue;
  const auto* d = static_cast<const AugDesc*>(descs);
  auto s = static_cast<cudaStream_t>(stream);
  if (n_stat > 0) {
    const long long blocks = 3LL * n_stat * slices;
    if (blocks > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
    histogram_kernel<<<(unsigned)blocks, kThreads, 0, s>>>(d, stat_images, scratch, slices);
    HB_LAUNCH_CHECK();
  }
  int rows_per_tile, tiles;
  if (!row_tiles<kThreads>(N, H, W, rows_per_tile, tiles)) return (int)cudaErrorInvalidValue;
  apply_kernel<<<(unsigned)(N * tiles), kThreads, 0, s>>>(d, params, scratch, slices, rows_per_tile, tiles);
  HB_LAUNCH_CHECK();
  return 0;
}
