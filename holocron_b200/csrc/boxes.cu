// Pairwise box operators (xyxy boxes, fp32 math): IoU, GIoU, DIoU penalty, DIoU/CIoU loss, aspect-ratio
// consistency, and the analytic backward of the IoU-based ones.
// Reference: holocron/ops/boxes.py:16-211 (+ torchvision.ops.boxes.box_iou). One launch per operator instead of
// ~30 tiny ATen kernels and 2 MxNx2 temporaries. The forward uses explicit round-to-nearest intrinsics in the
// reference's operation order (no FMA contraction) so the exact-value vectors of the reference's own tests
// (tests/test_ops.py:25-76) hold bit for bit.
//
// Also the box steps of the detection recipe's transforms (references/detection/transforms.py:58-127), every box of a
// batch in one launch (box_transform_kernel below), and the ground-truth matching of the detection trainer's evaluation
// (holocron/trainer/detection.py:17-32), every image of a batch in one launch (match_kernel below).
//
// NB (reference quirk, reproduced): ciou_loss adds its alpha*v term to a masked COPY (boxes.py:209), so it
// returns exactly the DIoU loss.
#include "common.cuh"

namespace {

enum Mode { M_IOU = 0, M_GIOU = 1, M_PENALTY = 2, M_DIOU_LOSS = 3, M_ARC = 4 };

struct Box { float x1, y1, x2, y2; };

__device__ __forceinline__ Box load_box(const float* p) { return Box{p[0], p[1], p[2], p[3]}; }

__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float dvd(float a, float b) { return __fdiv_rn(a, b); }

__device__ __forceinline__ void inter_union(const Box& a, const Box& b, float& inter, float& uni) {
  const float area_a = mul(sub(a.x2, a.x1), sub(a.y2, a.y1));
  const float area_b = mul(sub(b.x2, b.x1), sub(b.y2, b.y1));
  const float w = fmaxf(sub(fminf(a.x2, b.x2), fmaxf(a.x1, b.x1)), 0.f);
  const float h = fmaxf(sub(fminf(a.y2, b.y2), fmaxf(a.y1, b.y1)), 0.f);
  inter = mul(w, h);
  uni = sub(add(area_a, area_b), inter);
}

__device__ __forceinline__ float penalty(const Box& a, const Box& b) {
  const float cw = sub(fmaxf(a.x2, b.x2), fminf(a.x1, b.x1));
  const float ch = sub(fmaxf(a.y2, b.y2), fminf(a.y1, b.y1));
  const float c2 = add(mul(cw, cw), mul(ch, ch));
  const float dx = sub(add(a.x1, a.x2), add(b.x1, b.x2));
  const float dy = sub(add(a.y1, a.y2), add(b.y1, b.y2));
  const float r2 = dvd(add(mul(dx, dx), mul(dy, dy)), 4.f);
  return dvd(r2, c2);
}

__device__ __forceinline__ float pair_value(int mode, const Box& a, const Box& b) {
  float inter, uni;
  switch (mode) {
    case M_IOU:
      inter_union(a, b, inter, uni);
      return dvd(inter, uni);
    case M_GIOU: {
      inter_union(a, b, inter, uni);
      const float ew = fmaxf(sub(fmaxf(a.x2, b.x2), fminf(a.x1, b.x1)), 0.f);
      const float eh = fmaxf(sub(fmaxf(a.y2, b.y2), fminf(a.y1, b.y1)), 0.f);
      const float area = mul(ew, eh);
      return sub(dvd(inter, uni), dvd(sub(area, uni), area));
    }
    case M_PENALTY: return penalty(a, b);
    case M_DIOU_LOSS:
      inter_union(a, b, inter, uni);
      return add(sub(1.f, dvd(inter, uni)), penalty(a, b));
    case M_ARC: {
      const float va = atanf(dvd(sub(a.x2, a.x1), sub(a.y2, a.y1)));
      const float vb = atanf(dvd(sub(b.x2, b.x1), sub(b.y2, b.y1)));
      const float d = sub(va, vb);
      return mul(mul(d, d), 0.40528473456935105f);  // 4 / pi^2 rounded to fp32
    }
  }
  return 0.f;
}

// Tile = kRows rows of boxes1 x (blockDim.x * 4) columns of boxes2. A thread keeps its 4 boxes2 in registers, walks the
// rows (boxes1 row = one broadcast 16-byte load) and writes 4 consecutive outputs per row - one 128-bit store when the
// output row is 16-byte aligned. A 64-bit division and 8 scalar loads per PAIR would make this ALU bound. kMode is a template parameter so the per-pair switch is gone as well.
constexpr int kRows = 16;

template <int kMode>
__global__ void __launch_bounds__(128) pairwise_kernel(const float* __restrict__ b1, const float* __restrict__ b2,
                                                       float* __restrict__ out, int M, int N) {
  const int j0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (j0 >= N) return;
  const int i0 = blockIdx.y * kRows;
  const int i1 = min(i0 + kRows, M);
  Box b[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4 v = __ldg((const float4*)b2 + min(j0 + q, N - 1));
    b[q] = Box{v.x, v.y, v.z, v.w};
  }
  const bool vec = (N & 3) == 0 && j0 + 3 < N && ((size_t)out & 15) == 0;
  for (int i = i0; i < i1; ++i) {
    const float4 va = __ldg((const float4*)b1 + i);
    const Box a{va.x, va.y, va.z, va.w};
    float r[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) r[q] = pair_value(kMode, a, b[q]);
    float* o = out + (size_t)i * N + j0;
    if (vec) {
      *(float4*)o = make_float4(r[0], r[1], r[2], r[3]);
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (j0 + q < N) o[q] = r[q];
    }
  }
}

// degenerate-box flag for box_giou's AssertionError (any x2 < x1 or y2 < y1)
__global__ void degenerate_kernel(const float* __restrict__ b, int n, int* flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && (b[4 * i + 2] < b[4 * i] || b[4 * i + 3] < b[4 * i + 1])) atomicOr(flag, 1);
}

// ---- backward ---------------------------------------------------------------------------------------
// sub-gradients follow PyTorch: binary max/min split ties evenly, clamp(min=0) passes the gradient at 0.
__device__ __forceinline__ void dmax(float a, float b, float& da, float& db) {
  da = a > b ? 1.f : (a == b ? 0.5f : 0.f);
  db = 1.f - da;
}
__device__ __forceinline__ void dmin(float a, float b, float& da, float& db) {
  da = a < b ? 1.f : (a == b ? 0.5f : 0.f);
  db = 1.f - da;
}

// accumulates g * d value / d (a, b) into ga[4], gb[4]
__device__ __forceinline__ void pair_grad(int mode, const Box& a, const Box& b, float g, float* ga, float* gb) {
  const float wa = a.x2 - a.x1, ha = a.y2 - a.y1, wb = b.x2 - b.x1, hb_ = b.y2 - b.y1;
  const float ltx = fmaxf(a.x1, b.x1), lty = fmaxf(a.y1, b.y1), rbx = fminf(a.x2, b.x2), rby = fminf(a.y2, b.y2);
  const float wr = rbx - ltx, hr = rby - lty;
  const float w = fmaxf(wr, 0.f), h = fmaxf(hr, 0.f);
  const float inter = w * h;
  const float uni = wa * ha + wb * hb_ - inter;
  // coefficient of d inter, d area_a, d area_b in d value, plus enclosing-box terms
  float c_inter = 0.f, c_area = 0.f;  // d value = c_inter * d inter + c_area * (d area_a + d area_b) + ...
  float g_cw = 0.f, g_ch = 0.f;       // d value / d (enclosing width / height, unclamped)
  float g_dx = 0.f, g_dy = 0.f;       // d value / d (centre differences dx, dy)
  const float cwr = fmaxf(a.x2, b.x2) - fminf(a.x1, b.x1), chr = fmaxf(a.y2, b.y2) - fminf(a.y1, b.y1);
  if (mode == M_IOU || mode == M_GIOU || mode == M_DIOU_LOSS) {
    // iou = inter / uni, uni = area_a + area_b - inter
    const float s = (mode == M_DIOU_LOSS) ? -1.f : 1.f;
    c_inter += s * (uni + inter) / (uni * uni);
    c_area += s * (-inter / (uni * uni));
  }
  if (mode == M_GIOU) {
    // giou = iou - 1 + uni / area_c,  area_c = clamp(cw) * clamp(ch)
    const float cw = fmaxf(cwr, 0.f), ch = fmaxf(chr, 0.f);
    const float area_c = cw * ch;
    c_area += 1.f / area_c;
    c_inter += -1.f / area_c;
    const float g_area_c = -uni / (area_c * area_c);
    g_cw += g_area_c * ch * (cwr >= 0.f ? 1.f : 0.f);
    g_ch += g_area_c * cw * (chr >= 0.f ? 1.f : 0.f);
  }
  if (mode == M_PENALTY || mode == M_DIOU_LOSS) {
    const float c2 = cwr * cwr + chr * chr;
    const float dx = (a.x1 + a.x2) - (b.x1 + b.x2), dy = (a.y1 + a.y2) - (b.y1 + b.y2);
    const float r2 = (dx * dx + dy * dy) * 0.25f;
    g_dx += 0.5f * dx / c2;
    g_dy += 0.5f * dy / c2;
    const float g_c2 = -r2 / (c2 * c2);
    g_cw += g_c2 * 2.f * cwr;
    g_ch += g_c2 * 2.f * chr;
  }
  // chain to coordinates
  const float gi_w = c_inter * h * (wr >= 0.f ? 1.f : 0.f);  // d / d (rbx - ltx)
  const float gi_h = c_inter * w * (hr >= 0.f ? 1.f : 0.f);
  float da, db;
  float t[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // ax1 ay1 ax2 ay2 bx1 by1 bx2 by2
  dmax(a.x1, b.x1, da, db); t[0] -= gi_w * da; t[4] -= gi_w * db;   // ltx
  dmax(a.y1, b.y1, da, db); t[1] -= gi_h * da; t[5] -= gi_h * db;   // lty
  dmin(a.x2, b.x2, da, db); t[2] += gi_w * da; t[6] += gi_w * db;   // rbx
  dmin(a.y2, b.y2, da, db); t[3] += gi_h * da; t[7] += gi_h * db;   // rby
  // areas
  t[0] += c_area * (-ha); t[2] += c_area * ha; t[1] += c_area * (-wa); t[3] += c_area * wa;
  t[4] += c_area * (-hb_); t[6] += c_area * hb_; t[5] += c_area * (-wb); t[7] += c_area * wb;
  // enclosing box
  dmax(a.x2, b.x2, da, db); t[2] += g_cw * da; t[6] += g_cw * db;
  dmin(a.x1, b.x1, da, db); t[0] -= g_cw * da; t[4] -= g_cw * db;
  dmax(a.y2, b.y2, da, db); t[3] += g_ch * da; t[7] += g_ch * db;
  dmin(a.y1, b.y1, da, db); t[1] -= g_ch * da; t[5] -= g_ch * db;
  // centres
  t[0] += g_dx; t[2] += g_dx; t[4] -= g_dx; t[6] -= g_dx;
  t[1] += g_dy; t[3] += g_dy; t[5] -= g_dy; t[7] -= g_dy;
#pragma unroll
  for (int k = 0; k < 4; ++k) { ga[k] += g * t[k]; gb[k] += g * t[4 + k]; }
}

// thread r < M: gradient row of boxes1[r]; thread M + c: gradient row of boxes2[c]   (deterministic, no atomics)
__global__ void pairwise_bwd_kernel(const float* __restrict__ b1, const float* __restrict__ b2,
                                    const float* __restrict__ gout, float* __restrict__ g1, float* __restrict__ g2, int M,
                                    int N, int mode) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= M + N) return;
  float acc[4] = {0.f, 0.f, 0.f, 0.f}, dump[4] = {0.f, 0.f, 0.f, 0.f};
  if (t < M) {
    if (!g1) return;
    const Box a = load_box(b1 + 4 * t);
    for (int j = 0; j < N; ++j) pair_grad(mode, a, load_box(b2 + 4 * j), gout[(size_t)t * N + j], acc, dump);
#pragma unroll
    for (int k = 0; k < 4; ++k) g1[4 * t + k] = acc[k];
  } else {
    if (!g2) return;
    const int c = t - M;
    const Box b = load_box(b2 + 4 * c);
    for (int i = 0; i < M; ++i) pair_grad(mode, load_box(b1 + 4 * i), b, gout[(size_t)i * N + c], dump, acc);
#pragma unroll
    for (int k = 0; k < 4; ++k) g2[4 * c + k] = acc[k];
  }
}

// ---- detection transforms ----------------------------------------------------------------------------
// Reference: references/detection/transforms.py:58-127. The box steps of a transform chain are one op sequence shared
// by every image; each op reads its operands from the image's fp32 parameter row, in order. Every step rounds as the
// reference's separate torch ops round (one _rn intrinsic each, so no two steps contract into an FMA).
enum BoxOp {
  B_SCALE = 0,   // (sx, sy): x *= sx, y *= sy
  B_CLAMP = 1,   // (x_lo, x_hi, y_lo, y_hi): clamp, NaN kept as torch's clamp keeps it
  B_SUB = 2,     // (dx, dy): x -= dx, y -= dy
  B_FILTER = 3,  // (): drop the box when x1 == x2 or y1 == y2
  B_FLIP = 4,    // (flag, width): when flag != 0, (x1, x2) = (width - x2, width - x1)
  B_DIV = 5,     // (dx, dy): x /= dx, y /= dy
};

struct BoxDesc {
  long long boxes, labels, box_stride, label_stride, n, offset, unused0, unused1;
};

constexpr int kBoxWarps = 8;

__device__ __forceinline__ float clampf(float v, float lo, float hi) { return v != v ? v : fminf(fmaxf(v, lo), hi); }

// One warp per image walks its boxes 32 at a time; the survivors of each 32 are written after those of the previous
// ones (ballot + popc), so the image's boxes keep their order at its output offset. No atomics.
__global__ void __launch_bounds__(kBoxWarps * 32) box_transform_kernel(const BoxDesc* __restrict__ descs,
                                                                      const float* __restrict__ params,
                                                                      const int* __restrict__ ops, int n_ops,
                                                                      int n_params, int N, float* __restrict__ out_boxes,
                                                                      long long* __restrict__ out_labels,
                                                                      int* __restrict__ counts) {
  const int img = blockIdx.x * kBoxWarps + (int)(threadIdx.x >> 5);
  const unsigned lane = threadIdx.x & 31;
  if (img >= N) return;
  const BoxDesc d = descs[img];
  const float* src = reinterpret_cast<const float*>(d.boxes);
  const long long* lab = reinterpret_cast<const long long*>(d.labels);
  const float* p = params + (size_t)img * n_params;
  long long kept = 0;
  for (long long base = 0; base < d.n; base += 32) {
    const long long i = base + lane;
    bool keep = i < d.n;
    float x1 = 0.f, y1 = 0.f, x2 = 0.f, y2 = 0.f;
    long long label = 0;
    if (keep) {
      const float* b = src + i * d.box_stride;
      x1 = b[0], y1 = b[1], x2 = b[2], y2 = b[3];
      label = lab[i * d.label_stride];
    }
    for (int k = 0, q = 0; k < n_ops; ++k) {
      switch (__ldg(ops + k)) {
        case B_SCALE:
          x1 = mul(x1, p[q]), x2 = mul(x2, p[q]), y1 = mul(y1, p[q + 1]), y2 = mul(y2, p[q + 1]);
          q += 2;
          break;
        case B_CLAMP:
          x1 = clampf(x1, p[q], p[q + 1]), x2 = clampf(x2, p[q], p[q + 1]);
          y1 = clampf(y1, p[q + 2], p[q + 3]), y2 = clampf(y2, p[q + 2], p[q + 3]);
          q += 4;
          break;
        case B_SUB:
          x1 = sub(x1, p[q]), x2 = sub(x2, p[q]), y1 = sub(y1, p[q + 1]), y2 = sub(y2, p[q + 1]);
          q += 2;
          break;
        case B_FILTER:
          keep = keep && x1 != x2 && y1 != y2;
          break;
        case B_FLIP:
          if (p[q] != 0.f) {
            const float a = sub(p[q + 1], x2);
            x2 = sub(p[q + 1], x1);
            x1 = a;
          }
          q += 2;
          break;
        case B_DIV:
          x1 = dvd(x1, p[q]), x2 = dvd(x2, p[q]), y1 = dvd(y1, p[q + 1]), y2 = dvd(y2, p[q + 1]);
          q += 2;
          break;
      }
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    if (keep) {
      const long long o = d.offset + kept + __popc(ballot & ((1u << lane) - 1u));
      float* ob = out_boxes + 4 * o;
      ob[0] = x1, ob[1] = y1, ob[2] = x2, ob[3] = y2;
      out_labels[o] = label;
    }
    kept += __popc(ballot);
  }
  if (lane == 0) counts[img] = (int)kept;
}

// ---- detection evaluation: ground truth matched to predictions ---------------------------------------
// Reference: holocron/trainer/detection.py:17-32, as holocron_b200.trainer.assign_iou computes it on CUDA tensors: box_iou
// (pair_value's IoU), max(dim=1), values >= threshold, and of the kept targets claiming one prediction the one with the
// largest IoU (the lowest index on a tie) keeps it. One CTA per image.
enum LabelType { L_I64 = 0, L_I32 = 1 };

// codes: box dtypes (HB_DTYPE_*) and label types (LabelType), one byte each: gt boxes, pred boxes, gt labels, pred labels.
// Strides in elements. labels are 0 when the caller counts nothing.
struct MatchDesc {
  long long gt, pred, gt_labels, pred_labels, n_gt, n_pred, gt_rs, gt_cs, pred_rs, pred_cs, gt_ls, pred_ls, codes,
      offset, unused0, unused1;
};

constexpr int kMatchWarps = 8;
constexpr int kMatchRows = 4;      // ground-truth rows a warp holds in registers per pass
constexpr int kMatchTile = 1024;   // predictions staged in shared memory at a time (16 KB)

// Box i of a strided [n, 4] tensor, converted to fp32 as Tensor.float() converts it.
__device__ __forceinline__ Box load_box_any(long long base, long long i, long long rs, long long cs, int dtype) {
  switch (dtype) {
    case HB_DTYPE_BF16: {
      const __nv_bfloat16* p = reinterpret_cast<const __nv_bfloat16*>(base) + i * rs;
      return Box{__bfloat162float(p[0]), __bfloat162float(p[cs]), __bfloat162float(p[2 * cs]), __bfloat162float(p[3 * cs])};
    }
    case HB_DTYPE_F16: {
      const __half* p = reinterpret_cast<const __half*>(base) + i * rs;
      return Box{__half2float(p[0]), __half2float(p[cs]), __half2float(p[2 * cs]), __half2float(p[3 * cs])};
    }
    case HB_DTYPE_F64: {
      const double* p = reinterpret_cast<const double*>(base) + i * rs;
      return Box{__double2float_rn(p[0]), __double2float_rn(p[cs]), __double2float_rn(p[2 * cs]),
                 __double2float_rn(p[3 * cs])};
    }
    default: {
      const float* p = reinterpret_cast<const float*>(base) + i * rs;
      return Box{p[0], p[cs], p[2 * cs], p[3 * cs]};
    }
  }
}

__device__ __forceinline__ long long load_label(long long base, long long i, long long stride, int type) {
  return type == L_I32 ? (long long)reinterpret_cast<const int*>(base)[i * stride]
                       : reinterpret_cast<const long long*>(base)[i * stride];
}

// (va, ia) comes before (vb, ib) in torch's CUDA max(dim): NaN first, then the larger value, then the lower index.
// An index < 0 is "no candidate yet".
__device__ __forceinline__ bool beats(float va, int ia, float vb, int ib) {
  if (ib < 0) return ia >= 0;
  if (ia < 0) return false;
  if (va != va) return vb == vb || ia < ib;
  if (vb != vb) return false;
  return va > vb || (va == vb && ia < ib);
}

// scratch: (IoU bits, index) of every ground-truth row's maximum, 8 bytes per row at the image's offset. counts (or
// NULL): int64 {assigned, correct}, added to.
__global__ void __launch_bounds__(kMatchWarps * 32) match_kernel(const MatchDesc* __restrict__ descs, float thr,
                                                                 int2* scratch, long long* __restrict__ match,
                                                                 unsigned long long* __restrict__ counts) {
  __shared__ Box tile[kMatchTile];
  __shared__ unsigned long long red[2][kMatchWarps];
  const MatchDesc d = descs[blockIdx.x];
  const int warp = (int)(threadIdx.x >> 5), lane = (int)(threadIdx.x & 31);
  const int gt_dt = (int)(d.codes & 0xff), pred_dt = (int)((d.codes >> 8) & 0xff);
  int2* best = scratch + d.offset;
  // 1. every row's first maximal IoU: each lane walks its predictions in index order, then the warp merges the lanes
  for (long long g0 = 0; g0 < d.n_gt; g0 += kMatchWarps * kMatchRows) {
    Box a[kMatchRows];
    float bv[kMatchRows];
    int bi[kMatchRows];
#pragma unroll
    for (int r = 0; r < kMatchRows; ++r) {
      const long long g = g0 + warp + r * kMatchWarps;
      a[r] = g < d.n_gt ? load_box_any(d.gt, g, d.gt_rs, d.gt_cs, gt_dt) : Box{0.f, 0.f, 0.f, 0.f};
      bv[r] = 0.f;
      bi[r] = -1;
    }
    for (long long p0 = 0; p0 < d.n_pred; p0 += kMatchTile) {
      const int nt = (int)min((long long)kMatchTile, d.n_pred - p0);
      __syncthreads();
      for (int j = threadIdx.x; j < nt; j += kMatchWarps * 32) tile[j] = load_box_any(d.pred, p0 + j, d.pred_rs, d.pred_cs, pred_dt);
      __syncthreads();
      for (int j = lane; j < nt; j += 32) {
        const Box b = tile[j];
#pragma unroll
        for (int r = 0; r < kMatchRows; ++r) {
          float inter, uni;
          inter_union(a[r], b, inter, uni);
          const float v = dvd(inter, uni);
          if (beats(v, (int)p0 + j, bv[r], bi[r])) bv[r] = v, bi[r] = (int)p0 + j;
        }
      }
    }
#pragma unroll
    for (int r = 0; r < kMatchRows; ++r) {
#pragma unroll
      for (int s = 16; s > 0; s >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv[r], s);
        const int oi = __shfl_xor_sync(0xffffffffu, bi[r], s);
        if (beats(ov, oi, bv[r], bi[r])) bv[r] = ov, bi[r] = oi;
      }
      const long long g = g0 + warp + r * kMatchWarps;
      if (lane == 0 && g < d.n_gt) best[g] = make_int2(__float_as_int(bv[r]), bi[r]);
    }
  }
  __syncthreads();
  // 2. a kept row keeps its prediction unless another row claims it with a larger IoU, or an equal one at a lower index
  unsigned long long assigned = 0, correct = 0;
  const int gl_t = (int)((d.codes >> 16) & 0xff), pl_t = (int)((d.codes >> 24) & 0xff);
  for (long long g = threadIdx.x; g < d.n_gt; g += kMatchWarps * 32) {
    const int2 e = best[g];
    const float v = __int_as_float(e.x);
    bool keep = e.y >= 0 && v >= thr;
    for (long long o = 0; keep && o < d.n_gt; ++o) {
      const int2 f = best[o];
      const float w = __int_as_float(f.x);
      keep = !(f.y == e.y && (w > v || (w == v && o < g)));
    }
    match[d.offset + g] = keep ? e.y : -1;
    if (keep) {
      ++assigned;
      if (d.gt_labels && d.pred_labels)
        correct += load_label(d.gt_labels, g, d.gt_ls, gl_t) == load_label(d.pred_labels, e.y, d.pred_ls, pl_t);
    }
  }
  if (!counts) return;
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    assigned += __shfl_xor_sync(0xffffffffu, assigned, s);
    correct += __shfl_xor_sync(0xffffffffu, correct, s);
  }
  if (lane == 0) red[0][warp] = assigned, red[1][warp] = correct;
  __syncthreads();
  if (threadIdx.x == 0) {
    assigned = correct = 0;
#pragma unroll
    for (int w = 0; w < kMatchWarps; ++w) assigned += red[0][w], correct += red[1][w];
    if (assigned) atomicAdd(counts, assigned);
    if (correct) atomicAdd(counts + 1, correct);
  }
}

}  // namespace

extern "C" {

int hb_box_transform_batch(const void* descs, const float* params, const int* ops, int n_ops, int n_params, int N,
                           float* out_boxes, long long* out_labels, int* counts, void* stream) {
  if (N < 0 || n_ops < 0 || n_params < 0) return (int)cudaErrorInvalidValue;
  if (N == 0) return 0;
  const int blocks = (N + kBoxWarps - 1) / kBoxWarps;
  box_transform_kernel<<<blocks, kBoxWarps * 32, 0, (cudaStream_t)stream>>>(
      static_cast<const BoxDesc*>(descs), params, ops, n_ops, n_params, N, out_boxes, out_labels, counts);
  HB_LAUNCH_CHECK();
  return 0;
}

int hb_assign_iou_batch(const void* descs, int N, float iou_threshold, void* scratch, long long* match,
                        long long* counts, void* stream) {
  if (N < 0) return (int)cudaErrorInvalidValue;
  if (N == 0) return 0;
  match_kernel<<<N, kMatchWarps * 32, 0, (cudaStream_t)stream>>>(static_cast<const MatchDesc*>(descs), iou_threshold,
                                                                static_cast<int2*>(scratch), match,
                                                                reinterpret_cast<unsigned long long*>(counts));
  HB_LAUNCH_CHECK();
  return 0;
}

// mode: 0 IoU, 1 GIoU, 2 DIoU penalty (rho^2/c^2), 3 DIoU loss (= the reference's ciou_loss too), 4 aspect-ratio
// consistency. boxes: fp32 [M,4] / [N,4] xyxy contiguous; out: fp32 [M,N].
int hb_box_pairwise(const float* boxes1, const float* boxes2, float* out, int M, int N, int mode, void* stream) {
  const long long total = (long long)M * N;
  if (total == 0) return 0;
  if ((((size_t)boxes1) | ((size_t)boxes2)) & 15) return (int)cudaErrorMisalignedAddress;   // [*, 4] fp32 rows: float4 loads
  const dim3 grid((N + 4 * 128 - 1) / (4 * 128), (M + kRows - 1) / kRows);
  if (grid.y > 65535) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream;
  switch (mode) {
    case M_IOU: pairwise_kernel<M_IOU><<<grid, 128, 0, st>>>(boxes1, boxes2, out, M, N); break;
    case M_GIOU: pairwise_kernel<M_GIOU><<<grid, 128, 0, st>>>(boxes1, boxes2, out, M, N); break;
    case M_PENALTY: pairwise_kernel<M_PENALTY><<<grid, 128, 0, st>>>(boxes1, boxes2, out, M, N); break;
    case M_DIOU_LOSS: pairwise_kernel<M_DIOU_LOSS><<<grid, 128, 0, st>>>(boxes1, boxes2, out, M, N); break;
    case M_ARC: pairwise_kernel<M_ARC><<<grid, 128, 0, st>>>(boxes1, boxes2, out, M, N); break;
    default: return (int)cudaErrorInvalidValue;
  }
  HB_LAUNCH_CHECK();
  return 0;
}

// flag (device int, pre-zeroed) is set to 1 if any box has x2 < x1 or y2 < y1
int hb_box_degenerate(const float* boxes, int n, int* flag, void* stream) {
  if (n == 0) return 0;
  degenerate_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(boxes, n, flag);
  HB_LAUNCH_CHECK();
  return 0;
}

// gradients of sum(gout * op(boxes1, boxes2)) for modes 0-3; g1 [M,4] / g2 [N,4] may be NULL
int hb_box_pairwise_bwd(const float* boxes1, const float* boxes2, const float* gout, float* g1, float* g2, int M, int N,
                        int mode, void* stream) {
  if (mode == M_ARC) return (int)cudaErrorInvalidValue;
  if (M + N == 0) return 0;
  pairwise_bwd_kernel<<<(M + N + 127) / 128, 128, 0, (cudaStream_t)stream>>>(boxes1, boxes2, gout, g1, g2, M, N, mode);
  HB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
