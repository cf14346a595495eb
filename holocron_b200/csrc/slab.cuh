// Channel-slab geometry of the NHWC bf16 row-streaming kernels (bn_act.cu, se_gate.cu, dwconv.cu), their persistent
// grids and the fixed-order fold of their per-block channel sums.
// A block of kSlabThreads threads covers one slab of cg_t 8-channel groups x rows_t row lanes: thread (tx, ty) owns the 8
// consecutive channels (one 128-bit bf16 vector) of group tx on the rows of lane ty, so its per-channel values stay in
// registers while it walks the rows.
#pragma once
#include "common.cuh"

namespace hb {

constexpr int kSlabThreads = 256;

struct SlabGeo {
  int cg_total;  // C / 8
  int cg_t;      // channel groups per block (<= 32)
  int rows_t;    // row lanes per block
  int slabs;     // channel slabs (grid.y)
  __host__ static SlabGeo make(int C) {
    SlabGeo g;
    g.cg_total = C / 8;
    // balanced channel slabs: 38 groups -> 2 x 19 rather than 32 + 6 (the ragged last slab kept 80 % of its block's
    // threads idle on ReXNet's widths: 300, 366, 432, 576, ... channels)
    const int nslab = (g.cg_total + 31) / 32;
    g.cg_t = (g.cg_total + nslab - 1) / nslab;
    g.rows_t = kSlabThreads / g.cg_t;
    g.slabs = (g.cg_total + g.cg_t - 1) / g.cg_t;
    return g;
  }
  // most row blocks (grid.x) when the grid holds per_sm blocks per SM over all slabs
  __host__ int max_blocks(int per_sm) const {
    const int cap = (HB_NUM_SMS * per_sm) / slabs;
    return cap < 1 ? 1 : cap;
  }
  // persistent grid (row blocks x slabs), grid-stride over `items` with `lanes` items per block and step: at least
  // ~min_rows items per lane when there is enough work, at most max_blocks(per_sm) row blocks
  __host__ dim3 grid(long long items, int per_sm, int min_rows, int lanes) const {
    const long long row_blocks = (items + lanes - 1) / lanes, cap = max_blocks(per_sm);
    long long want = (row_blocks + min_rows - 1) / min_rows;
    if (want < 1) want = 1;
    if (want > cap) want = cap;
    return dim3((unsigned)want, (unsigned)slabs);
  }
  // one item per row lane
  __host__ dim3 grid(long long items, int per_sm, int min_rows = 4) const { return grid(items, per_sm, min_rows, rows_t); }
  // this thread's channel group tx inside the slab, row lane ty, global channel group cg, and whether it streams rows (a
  // spare lane or a group past the last one streams nothing but still has to reach the block's barriers)
  struct Thread {
    int tx, ty, cg;
    bool active;
  };
  __device__ __forceinline__ Thread thread() const {
    const int tx = threadIdx.x % cg_t, ty = threadIdx.x / cg_t;
    const int cg = blockIdx.y * cg_t + tx;
    return {tx, ty, cg, ty < rows_t && cg < cg_total};
  }
};

// Block fold of NS per-channel sums: every thread has left its 8 per-channel values of sum s at red[s][threadIdx.x * 8 ...]
// (red = [NS][kSlabThreads * 8] floats in shared memory, written before a __syncthreads). Threads 0 .. cg_t*8-1 each own one
// channel of the slab and add its rows_t lane values in lane order in Acc (a fixed order: run-to-run identical), then call
// emit(c, sums) with the channel c and its NS sums.
template <typename Acc, int NS, typename Emit>
__device__ __forceinline__ void fold_row_lanes(const SlabGeo& g, const float* red, Emit emit) {
  const int nch = g.cg_t * 8;
  for (int ch = threadIdx.x; ch < nch; ch += kSlabThreads) {
    const int ctx = ch / 8, j = ch % 8;
    const int gcg = blockIdx.y * g.cg_t + ctx;
    if (gcg >= g.cg_total) continue;
    Acc a[NS];
#pragma unroll
    for (int s = 0; s < NS; ++s) a[s] = Acc(0);
    for (int r = 0; r < g.rows_t; ++r) {
#pragma unroll
      for (int s = 0; s < NS; ++s) a[s] += (Acc)red[s * kSlabThreads * 8 + (r * g.cg_t + ctx) * 8 + j];
    }
    emit(gcg * 8 + j, a);
  }
}

}  // namespace hb
