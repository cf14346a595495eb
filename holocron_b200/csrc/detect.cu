// YOLO inference post-processing for a whole batch: select, order, suppress, emit.
// Reference: holocron/models/detection/yolo.py:159-233 (YOLOv1 / YOLOv2 post_process) and yolov4.py:303-335 (YoloLayer
// post_process, concatenated per image by the head). The reference loops over images in Python: per image a host
// synchronisation on `torch.any`, two or three boolean-mask gathers and a torchvision `nms`. Here every (image, segment)
// pair of a batch goes through one chain of five launches with no host synchronisation and no atomics:
//
//   1. select_kernel   a thread per candidate: score = first max over the classes x objectness; kept when objectness
//                      >= 0.5 and score >= the segment's threshold. Writes a 32-bit sort key (or a reject sentinel).
//   2. order_kernel    a CTA per (image, segment): block prefix scan of the kept flags in candidate order (the order
//                      of the reference's boolean masks), then a bitonic sort of (score descending, candidate index)
//                      keys - a stable descending sort, the tie rule of torchvision's CUDA nms - in shared memory for a
//                      segment of up to kSmemKeys candidates, in global scratch for a larger one. Writes the survivors' clamped boxes, scores and
//                      labels in score order.
//   3. mask_kernel     a CTA per (64-box row block, image, segment): bit j of word (row, j / 64) is set when
//                      IoU(row, j) > threshold for j > row, with torchvision's sm_90 arithmetic (see iou_above).
//   4. walk_kernel     a CTA per (image, segment) walks the mask in score order, 64 boxes per step, and lists the kept
//                      boxes.
//   5. emit_kernel     a thread per output slot: concatenates the kept boxes of an image's segments in segment order
//                      into the padded outputs, zero-fills the tail and writes the per-image count.
//
// The clamp to [0, 1] is applied once: clamp(clamp(x)) == clamp(x) bit for bit, so YOLOv1/v2's "clamp, then mask" and
// YOLOv4's "clamp, mask, clamp again" give the same boxes.
#include "common.cuh"
#include "holocron_b200.h"

namespace {

constexpr int kMaxSegs = 4;
constexpr int kSmemKeys = 16384;          // 128 KiB of 64-bit keys: one segment of up to 16384 candidates sorts in smem
constexpr int kOrderThreads = 512;
constexpr int kWalkThreads = 256;
constexpr int kMaxCandidates = 1 << 20;   // per image and segment: the walk's removed-bit words fit in 128 KiB
constexpr unsigned kReject = 0xFFFFFFFFu;  // never the key of a kept score: only a NaN maps there, and NaN is not kept

struct Seg {
  const float* boxes;   // [B, M, 4]
  const float* obj;     // [B, M]
  const float* cls;     // [B, M, K]
  int M, nb;            // candidates per image, 64-box blocks per image
  float score_thresh, iou_thresh;
  long long cand_off;   // B * (candidates of the earlier segments): start of this segment in the per-candidate arrays
  long long mask_off;   // start of this segment's bitmask words
};

struct Params {
  Seg seg[kMaxSegs];
  int nseg, B, K, cap;
  unsigned* key;         // [N] per candidate
  float* score;          // [N]
  int* label;            // [N]
  float4* sbox;          // [N] survivors in score order
  float* sscore;         // [N]
  int* slabel;           // [N]
  int* keep;             // [N] kept positions (indices into the sorted survivors)
  int* count;            // [B * nseg] survivors
  int* kept;             // [B * nseg] kept boxes
  unsigned long long* mask;
  unsigned long long* gkeys;   // [B * nseg * pkeys] when pkeys > kSmemKeys, used by the segments with M > kSmemKeys
  int pkeys;             // keys per (image, segment) sort: next power of two of the largest M
};

// the segment's fields in registers (a dynamically indexed kernel parameter would be copied to local memory)
__device__ __forceinline__ Seg seg_of(const Params& p, int s) {
  Seg r = p.seg[0];
#pragma unroll
  for (int t = 1; t < kMaxSegs; ++t)
    if (t == s) r = p.seg[t];
  return r;
}

__device__ __forceinline__ float clamp01(float x) { return x != x ? x : fminf(fmaxf(x, 0.f), 1.f); }

// score -> key that sorts ascending in descending score order; -0 and +0 compare equal, as in a comparison sort
__device__ __forceinline__ unsigned desc_key(float s) {
  const unsigned u = __float_as_uint(s == 0.f ? 0.f : s);
  const unsigned asc = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ~asc;
}

// torchvision's devIoU as ptxas compiles it for sm_90 (nms_kernel_impl<float> in torchvision 0.26): the first box's
// area is a plain product, the second box's area is fused into the sum (one FFMA), then inter is subtracted, an IEEE
// division and a strict comparison. Same operations, same rounding: every decision matches bit for bit.
__device__ __forceinline__ bool iou_above(float4 a, float area_a, float4 b, float thr) {
  const float sum = __fmaf_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y), area_a);
  const float w = fmaxf(__fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x)), 0.f);
  const float h = fmaxf(__fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y)), 0.f);
  const float inter = __fmul_rn(w, h);
  return __fdiv_rn(inter, __fsub_rn(sum, inter)) > thr;
}

__global__ void __launch_bounds__(256) select_kernel(Params p) {
  const int g = blockIdx.y, s = g % p.nseg, b = g / p.nseg;
  const Seg sg = seg_of(p, s);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= sg.M) return;
  const long long c = (long long)b * sg.M + i;
  const float* cl = sg.cls + c * p.K;
  float best = cl[0];
  int lab = 0;
  for (int k = 1; k < p.K; ++k) {
    const float v = cl[k];
    if (v > best || (v != v && best == best)) { best = v; lab = k; }   // first maximum, NaN wins (torch's max)
  }
  const float o = sg.obj[c];
  const float score = __fmul_rn(best, o);
  const long long at = sg.cand_off + c;
  p.key[at] = (o >= 0.5f && score >= sg.score_thresh) ? desc_key(score) : kReject;
  p.score[at] = score;
  p.label[at] = lab;
}

__global__ void __launch_bounds__(kOrderThreads) order_kernel(Params p) {
  extern __shared__ unsigned long long smem_keys[];
  __shared__ int warp_sum[kOrderThreads / 32];
  __shared__ int total;
  const int g = blockIdx.x, s = g % p.nseg, b = g / p.nseg;
  const Seg sg = seg_of(p, s);
  const long long base = sg.cand_off + (long long)b * sg.M;
  // each segment sorts in shared memory when its own candidates fit there, in global scratch otherwise
  unsigned long long* keys = sg.M > kSmemKeys ? p.gkeys + (long long)g * p.pkeys : smem_keys;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // compaction in candidate order: block prefix scan of the kept flags, chunk by chunk
  int n = 0;
  for (int start = 0; start < sg.M; start += kOrderThreads) {
    const int i = start + tid;
    const unsigned k = i < sg.M ? p.key[base + i] : kReject;
    const bool f = k != kReject;
    const unsigned bal = __ballot_sync(0xffffffffu, f);
    if (lane == 0) warp_sum[warp] = __popc(bal);
    __syncthreads();
    if (warp == 0) {
      constexpr int kWarps = kOrderThreads / 32;
      const int v = lane < kWarps ? warp_sum[lane] : 0;
      int incl = v;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += t;
      }
      if (lane < kWarps) warp_sum[lane] = incl - v;
      if (lane == 31) total = incl;
    }
    __syncthreads();
    if (f) keys[n + warp_sum[warp] + __popc(bal & ((1u << lane) - 1u))] = ((unsigned long long)k << 32) | (unsigned)i;
    n += total;
    __syncthreads();
  }
  int pn = 1;
  while (pn < n) pn <<= 1;
  for (int i = n + tid; i < pn; i += kOrderThreads) keys[i] = ~0ull;
  __syncthreads();
  // bitonic sort, ascending keys = descending scores, equal scores by candidate index
  for (int k = 2; k <= pn; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = tid; t < (pn >> 1); t += kOrderThreads) {
        const int i = 2 * j * (t / j) + (t % j);
        const int l = i + j;
        const unsigned long long x = keys[i], y = keys[l];
        if ((x > y) == ((i & k) == 0)) { keys[i] = y; keys[l] = x; }
      }
      __syncthreads();
    }
  }
  for (int r = tid; r < n; r += kOrderThreads) {
    const int i = (int)(keys[r] & 0xFFFFFFFFu);
    const float4 v = __ldg(reinterpret_cast<const float4*>(sg.boxes) + (long long)b * sg.M + i);
    p.sbox[base + r] = make_float4(clamp01(v.x), clamp01(v.y), clamp01(v.z), clamp01(v.w));
    p.sscore[base + r] = p.score[base + i];
    p.slabel[base + r] = p.label[base + i];
  }
  if (tid == 0) p.count[g] = n;
}

__global__ void __launch_bounds__(64) mask_kernel(Params p) {
  __shared__ float4 cols[64];
  const int g = blockIdx.y, s = g % p.nseg, b = g / p.nseg;
  const Seg sg = seg_of(p, s);
  const int n = p.count[g];
  const int rb = blockIdx.x;
  if (rb * 64 >= n) return;
  const long long base = sg.cand_off + (long long)b * sg.M;
  const int tid = threadIdx.x, row = rb * 64 + tid;
  const float4 a = row < n ? p.sbox[base + row] : make_float4(0.f, 0.f, 0.f, 0.f);
  const float area_a = __fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y));
  unsigned long long* mrow = p.mask + sg.mask_off + ((long long)b * sg.M + row) * sg.nb;
  const int nbc = (n + 63) / 64;
  for (int jb = rb; jb < nbc; ++jb) {
    const int col = jb * 64 + tid;
    cols[tid] = col < n ? p.sbox[base + col] : make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    if (row < n) {
      const int lim = min(64, n - jb * 64);
      unsigned long long bits = 0;
      for (int i = jb == rb ? tid + 1 : 0; i < lim; ++i)
        if (iou_above(a, area_a, cols[i], sg.iou_thresh)) bits |= 1ull << i;
      mrow[jb] = bits;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kWalkThreads) walk_kernel(Params p) {
  extern __shared__ unsigned long long removed[];
  __shared__ unsigned long long keep_bits;
  const int g = blockIdx.x, s = g % p.nseg, b = g / p.nseg;
  const Seg sg = seg_of(p, s);
  const int n = p.count[g];
  const int nbc = (n + 63) / 64;
  const long long base = sg.cand_off + (long long)b * sg.M;
  const unsigned long long* mimg = p.mask + sg.mask_off + (long long)b * sg.M * sg.nb;
  const int tid = threadIdx.x, lane = tid & 31;
  for (int w = tid; w < nbc; w += kWalkThreads) removed[w] = 0;
  __syncthreads();
  int kept = 0;
  for (int jb = 0; jb < nbc; ++jb) {
    const int lim = min(64, n - jb * 64);
    if (tid < 32) {
      // rows jb*64 + lane and jb*64 + 32 + lane: their words on the diagonal block
      const unsigned long long d0 = lane < lim ? mimg[(long long)(jb * 64 + lane) * sg.nb + jb] : 0;
      const unsigned long long d1 = lane + 32 < lim ? mimg[(long long)(jb * 64 + 32 + lane) * sg.nb + jb] : 0;
      const unsigned long long valid = lim == 64 ? ~0ull : (1ull << lim) - 1;
      unsigned long long word = removed[jb], kb = 0;
      unsigned long long avail = ~word & valid;
      while (avail) {                     // uniform across the warp: word and kb are the same in every lane
        const int i = __ffsll((long long)avail) - 1;
        kb |= 1ull << i;
        word |= __shfl_sync(0xffffffffu, i < 32 ? d0 : d1, i & 31);
        avail = ~word & valid & (~0ull << i << 1);
      }
      if (lane == 0) keep_bits = kb;
    }
    __syncthreads();
    const unsigned long long kb = keep_bits;
    for (int r = tid; r < 64; r += kWalkThreads)
      if ((kb >> r) & 1) p.keep[base + kept + __popcll(kb & ((1ull << r) - 1))] = jb * 64 + r;
    for (int w = jb + 1 + tid; w < nbc; w += kWalkThreads) {
      unsigned long long acc = removed[w];
      for (unsigned long long t = kb; t; t &= t - 1)
        acc |= mimg[(long long)(jb * 64 + __ffsll((long long)t) - 1) * sg.nb + w];
      removed[w] = acc;
    }
    kept += __popcll(kb);
    __syncthreads();
  }
  if (tid == 0) p.kept[g] = kept;
}

__global__ void __launch_bounds__(256) emit_kernel(Params p, float* __restrict__ out_boxes, float* __restrict__ out_scores,
                                                   long long* __restrict__ out_labels, int* __restrict__ counts) {
  const int b = blockIdx.y;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= max(p.cap, 1)) return;
  int total = 0, src = -1;
  long long base = 0;
  for (int s = 0; s < p.nseg; ++s) {
    const int k = p.kept[b * p.nseg + s];
    if (src < 0 && q < total + k) {
      base = p.seg[s].cand_off + (long long)b * p.seg[s].M;
      src = p.keep[base + q - total];
    }
    total += k;
  }
  if (q == 0) counts[b] = total;
  if (q >= p.cap) return;
  const long long o = (long long)b * p.cap + q;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  float sc = 0.f;
  long long lab = 0;
  if (src >= 0) {
    v = p.sbox[base + src];
    sc = p.sscore[base + src];
    lab = p.slabel[base + src];
  }
  reinterpret_cast<float4*>(out_boxes)[o] = v;
  out_scores[o] = sc;
  out_labels[o] = lab;
}

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// Fills p's segment table and scratch pointers (scratch may be NULL: sizing only). Returns the scratch size, or 0 for
// an invalid table.
size_t plan(const hb_detect_seg* segs, int nseg, int B, int K, char* scratch, Params& p) {
  if (!segs || nseg < 1 || nseg > kMaxSegs || B < 0 || K < 1) return 0;
  p = Params{};
  p.nseg = nseg; p.B = B; p.K = K;
  long long mtot = 0, mask_words = 0;
  int mmax = 0;
  for (int s = 0; s < nseg; ++s) {
    const int M = segs[s].M;
    if (M < 0 || M > kMaxCandidates) return 0;
    Seg& sg = p.seg[s];
    sg.boxes = segs[s].boxes; sg.obj = segs[s].obj; sg.cls = segs[s].cls;
    sg.M = M; sg.nb = (M + 63) / 64;
    sg.score_thresh = segs[s].score_thresh; sg.iou_thresh = segs[s].iou_thresh;
    sg.cand_off = (long long)B * mtot;
    sg.mask_off = mask_words;
    mtot += M;
    mask_words += (long long)B * M * sg.nb;
    mmax = M > mmax ? M : mmax;
  }
  if (mtot > 0x7FFFFFFF || (long long)B * nseg > 65535) return 0;
  p.cap = (int)mtot;
  int pk = 1;
  while (pk < mmax) pk <<= 1;
  p.pkeys = pk;
  const long long N = (long long)B * mtot;
  size_t off = 0;
  auto take = [&](size_t bytes) { char* at = scratch ? scratch + off : nullptr; off += align256(bytes); return at; };
  p.key = (unsigned*)take(N * 4);
  p.score = (float*)take(N * 4);
  p.label = (int*)take(N * 4);
  p.sbox = (float4*)take(N * 16);
  p.sscore = (float*)take(N * 4);
  p.slabel = (int*)take(N * 4);
  p.keep = (int*)take(N * 4);
  p.count = (int*)take((size_t)B * nseg * 4);
  p.kept = (int*)take((size_t)B * nseg * 4);
  p.mask = (unsigned long long*)take(mask_words * 8);
  p.gkeys = (unsigned long long*)take(pk > kSmemKeys ? (size_t)B * nseg * pk * 8 : 0);
  return off == 0 ? 1 : off;
}

}  // namespace

extern "C" {

size_t hb_detect_scratch_bytes(const hb_detect_seg* segs, int nseg, int B, int K) {
  Params p;
  return plan(segs, nseg, B, K, nullptr, p);
}

int hb_detect(const hb_detect_seg* segs, int nseg, int B, int K, void* scratch, float* out_boxes, float* out_scores,
              long long* out_labels, int* counts, void* stream) {
  Params p;
  if (plan(segs, nseg, B, K, (char*)scratch, p) == 0) return (int)cudaErrorInvalidValue;
  if (B == 0) return 0;
  if (((size_t)out_boxes & 15) || ((size_t)scratch & 255)) return (int)cudaErrorMisalignedAddress;
  int mmax = 0;
  for (int s = 0; s < nseg; ++s) {
    if (((size_t)segs[s].boxes & 15) || (segs[s].M > 0 && (!segs[s].boxes || !segs[s].obj || !segs[s].cls)))
      return (int)cudaErrorInvalidValue;
    mmax = segs[s].M > mmax ? segs[s].M : mmax;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int G = B * nseg;
  const int nbmax = (mmax + 63) / 64;
  if (mmax > 0) {
    select_kernel<<<dim3((mmax + 255) / 256, G), 256, 0, st>>>(p);
    HB_LAUNCH_CHECK();
    const size_t order_smem = (size_t)(p.pkeys < kSmemKeys ? p.pkeys : kSmemKeys) * 8;
    if (order_smem > 48 * 1024)
      cudaFuncSetAttribute(order_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)order_smem);
    order_kernel<<<G, kOrderThreads, order_smem, st>>>(p);
    HB_LAUNCH_CHECK();
    mask_kernel<<<dim3(nbmax, G), 64, 0, st>>>(p);
    HB_LAUNCH_CHECK();
  } else {
    cudaMemsetAsync(p.count, 0, (size_t)G * 4, st);
  }
  const size_t walk_smem = (size_t)(nbmax > 0 ? nbmax : 1) * 8;
  if (walk_smem > 48 * 1024)
    cudaFuncSetAttribute(walk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)walk_smem);
  walk_kernel<<<G, kWalkThreads, walk_smem, st>>>(p);
  HB_LAUNCH_CHECK();
  emit_kernel<<<dim3((p.cap > 0 ? p.cap + 255 : 256) / 256, B), 256, 0, st>>>(p, out_boxes, out_scores, out_labels,
                                                                              counts);
  HB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
