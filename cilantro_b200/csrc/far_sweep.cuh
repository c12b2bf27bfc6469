// Far-query path of the grid searches (product code, sm_90a).
// The shell sweeps of nn_search.cuh / grid_sweep.cuh cost O(k^2) row tests for shell k whether or not the
// shell holds points, so a query that has to cross a lot of empty space (a point far outside the cloud, the
// centre of a hollow scan, an isolated outlier asking for k neighbours) would spend O(k^3) on nothing. Once a
// sweep has used up its row budget it restarts here: the grid's list of NON-EMPTY coarse blocks (8^3 cells,
// GridView::blocks) is walked instead, every block pruned by a conservative lower bound of its distance.
//   1. radius bound R: the smallest block "far corner" distance within which the blocks are known to hold at
//      least k_needed points (every non-empty block has >= 1 point inside its box) — so the k_needed nearest
//      points have d2 <= R;
//   2. walk: blocks with lower bound > R or >= bound() are skipped, the others are scanned row by row with
//      the same row pruning and the same scan() as the shell sweeps.
// Exactness: a skipped block cannot hold a point that belongs to the result (distance bounds use the same
// 2^-10-cell margin and hs2 as nn_search.cuh; upper bounds are inflated the same way), and the candidate
// handling (strict d2 < bound, ties on the original index) is the caller's scan(), unchanged. The walk visits
// every candidate at most once, so callers reset their result before calling far_sweep.
//
// Included by nn_search.cuh (after cell_coord / slab_gap / kCellMargin); do not include directly.
#pragma once

namespace cb {

constexpr int kFarRowBudget = 6000;  // row tests a shell sweep may spend before it switches to the block walk

struct BlockBounds {
  float lo2;  // lower bound of d2 / h^2 to any point of the block (cells^2, margin applied)
  float hi2;  // upper bound of d2 / h^2 to every point of the block (cells^2, margin applied)
};

__device__ __forceinline__ BlockBounds block_bounds(const uint4 b, float fx, float fy, float fz, int nx, int ny,
                                                    int nz) {
  const float x0 = (float)(b.x * kBlockCells), x1 = (float)min((int)(b.x + 1) * kBlockCells, nx);
  const float y0 = (float)(b.y * kBlockCells), y1 = (float)min((int)(b.y + 1) * kBlockCells, ny);
  const float z0 = (float)(b.z * kBlockCells), z1 = (float)min((int)(b.z + 1) * kBlockCells, nz);
  auto gap = [](float f, float a0, float a1) {
    float g = fmaxf(fmaxf(a0 - f, f - a1), 0.f) - kCellMargin;
    return g > 0.f ? g : 0.f;
  };
  auto reach = [](float f, float a0, float a1) { return fmaxf(fabsf(f - a0), fabsf(a1 - f)) + kCellMargin; };
  const float gx = gap(fx, x0, x1), gy = gap(fy, y0, y1), gz = gap(fz, z0, z1);
  const float rx = reach(fx, x0, x1), ry = reach(fy, y0, y1), rz = reach(fz, z0, z1);
  BlockBounds r;
  r.lo2 = gx * gx + gy * gy + gz * gz;
  r.hi2 = rx * rx + ry * ry + rz * rz;
  return r;
}

// Smallest upper bound R2 (world units, inflated) such that the blocks with hi2 <= R2 hold >= k_needed points;
// +inf when the cloud has fewer points or k_needed == 0.
__device__ __forceinline__ float far_radius_bound(const GridView& g, float fx, float fy, float fz, uint32_t k_needed,
                                                  float h_up2) {
  const float inf = __int_as_float(0x7f800000);
  if (k_needed == 0 || g.n < k_needed) return inf;
  float r = inf;
  for (uint32_t i = 0; i < g.nblocks; ++i) r = fminf(r, block_bounds(__ldg(g.blocks + i), fx, fy, fz, g.nx, g.ny, g.nz).hi2);
  if (k_needed > 1) {
    // grow until enough points are certainly inside: at most ~log2(extent^2) rounds for a finite query; the
    // round cap makes a NaN / Inf query (all comparisons false) fall back to "no bound" instead of spinning
    bool enough = false;
    for (int round = 0; round < 96 && !enough; ++round) {
      uint32_t c = 0;
      for (uint32_t i = 0; i < g.nblocks; ++i) {
        const uint4 b = __ldg(g.blocks + i);
        if (block_bounds(b, fx, fy, fz, g.nx, g.ny, g.nz).hi2 <= r) c += b.w;
      }
      enough = c >= k_needed;
      if (!enough) r *= 2.f;
    }
    if (!enough) return inf;
  }
  return r * h_up2;
}

template <class BoundFn, class ScanFn>
__device__ __forceinline__ void far_sweep(const GridView& g, float qx, float qy, float qz, uint32_t k_needed,
                                          BoundFn bound, ScanFn scan) {
  const float fx = cell_coord(qx, g.ox, g.inv_h), fy = cell_coord(qy, g.oy, g.inv_h),
              fz = cell_coord(qz, g.oz, g.inv_h);
  const int cy = (int)floorf(fy), cz = (int)floorf(fz);
  const float hs2 = g.hs2;
  const float h_up = g.h_safe * 1.00390625f;  // >= h (1 + 2^-10): h_safe = h (1 - 2^-10)
  const float r2 = far_radius_bound(g, fx, fy, fz, k_needed, h_up * h_up);
  for (uint32_t i = 0; i < g.nblocks; ++i) {
    const uint4 b = __ldg(g.blocks + i);
    const float lo = block_bounds(b, fx, fy, fz, g.nx, g.ny, g.nz).lo2 * hs2;
    if (lo > r2 || lo > bound()) continue;
    const int x0 = (int)b.x * kBlockCells, x1 = min(x0 + kBlockCells, g.nx);
    const int ye = min((int)(b.y + 1) * kBlockCells, g.ny), ze = min((int)(b.z + 1) * kBlockCells, g.nz);
    for (int rz = (int)b.z * kBlockCells; rz < ze; ++rz) {
      const float gz = slab_gap(fz, cz, rz);
      const float gz2 = gz * gz;
      if (gz2 * hs2 > bound()) continue;
      for (int ry = (int)b.y * kBlockCells; ry < ye; ++ry) {
        const float gy = slab_gap(fy, cy, ry);
        if ((gy * gy + gz2) * hs2 > bound()) continue;
        const uint32_t base = ((uint32_t)rz * (uint32_t)g.ny + (uint32_t)ry) * (uint32_t)g.nx;
        const uint32_t s = __ldg(g.cell_start + base + x0), e = __ldg(g.cell_start + base + x1);
        if (s < e) scan(s, e);
      }
    }
  }
}

}  // namespace cb
