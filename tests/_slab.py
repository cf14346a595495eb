"""Python mirror of the channel-slab geometry of csrc/slab.cuh (``SlabGeo::make``, ``max_blocks`` and ``grid``), which
the BatchNorm, squeeze-excite and depth-wise convolution kernels share (no GPU). The SM count sizes the grids, so the
grid helpers take it as an argument (H100 SXM: 132, H100 PCIe: 114)."""
from typing import NamedTuple, Optional


class Geo(NamedTuple):
    cg_total: int   # 8-channel groups
    slabs: int      # channel slabs (grid.y)
    cg_t: int       # groups per slab
    rows_t: int     # row lanes per block


def geometry(c: int) -> Geo:
    """Balanced channel slabs of at most 32 groups of 8 channels, the rest of the 256 threads as row lanes."""
    cg_total = c // 8
    slabs = -(-cg_total // 32)
    cg_t = -(-cg_total // slabs)
    return Geo(cg_total, slabs, cg_t, 256 // cg_t)


def max_blocks(c: int, sms: int, per_sm: int) -> int:
    """Most row blocks of a grid of ``per_sm`` blocks per SM over all slabs."""
    return max((sms * per_sm) // geometry(c).slabs, 1)


def grid_rows(c: int, m: int, sms: int, per_sm: int, min_rows: int = 4, lanes: Optional[int] = None) -> int:
    """grid.x (row blocks) of SlabGeo::grid over ``m`` items, ``lanes`` of them per block and step (default rows_t)."""
    lanes = geometry(c).rows_t if lanes is None else lanes
    row_blocks = -(-m // lanes)
    return max(min(-(-row_blocks // min_rows), max_blocks(c, sms, per_sm)), 1)
