// Generic shell sweep over the uniform grid (product code, sm_90a): visits, for one query, every cell
// range that can still hold a point closer than bound(), in growing Chebyshev shells around the query's
// cell, with the same conservative pruning as nn_search.cuh (2^-10 cell margin, hs2). bound() may
// shrink while scanning (k-best lists) or stay constant (radius neighbourhoods).
//   bound(): float      current admissible squared distance (strict: candidates need d2 < bound)
//   scan(b, e)          consume the cell-sorted points [b, e)
//   reset()             forget everything consumed so far (the sweep restarts on the far-query path,
//                       far_sweep.cuh, when crossing empty space shell by shell gets too expensive)
//   k_needed            how many neighbours the caller is after (0 = all within a fixed bound)
#pragma once
#include "nn_search.cuh"

namespace cb {

template <class BoundFn, class ScanFn, class ResetFn>
__device__ __forceinline__ void grid_sweep(const GridView& g, float qx, float qy, float qz, BoundFn bound,
                                           ScanFn scan, ResetFn reset, uint32_t k_needed) {
  if (g.n == 0) return;
  // a NaN / Inf query is at no finite distance from anything: no candidate can pass d2 < bound
  if (!(fabsf(qx) + fabsf(qy) + fabsf(qz) < 3.0e38f)) return;
  const float fx = cell_coord(qx, g.ox, g.inv_h), fy = cell_coord(qy, g.oy, g.inv_h),
              fz = cell_coord(qz, g.oz, g.inv_h);
  const int cx = (int)floorf(fx), cy = (int)floorf(fy), cz = (int)floorf(fz);
  const float hs2 = g.hs2;
  int k0 = 0;
  k0 = max(k0, cx < 0 ? -cx : (cx > g.nx - 1 ? cx - (g.nx - 1) : 0));
  k0 = max(k0, cy < 0 ? -cy : (cy > g.ny - 1 ? cy - (g.ny - 1) : 0));
  k0 = max(k0, cz < 0 ? -cz : (cz > g.nz - 1 ? cz - (g.nz - 1) : 0));
  int row_budget = kFarRowBudget;
  for (int sh = k0;; ++sh) {
    if (sh > 0) {
      // termination: distance to the nearest unscanned face vs the bound (a point beyond the face
      // has a d2 strictly greater than the bound, so it cannot enter even on a tie)
      const int kk = sh - 1;
      float cover = 3.0e38f;
      bool any = false;
      if (cx - kk > 0) { cover = fminf(cover, fx - (float)(cx - kk)); any = true; }
      if (cx + kk < g.nx - 1) { cover = fminf(cover, (float)(cx + kk + 1) - fx); any = true; }
      if (cy - kk > 0) { cover = fminf(cover, fy - (float)(cy - kk)); any = true; }
      if (cy + kk < g.ny - 1) { cover = fminf(cover, (float)(cy + kk + 1) - fy); any = true; }
      if (cz - kk > 0) { cover = fminf(cover, fz - (float)(cz - kk)); any = true; }
      if (cz + kk < g.nz - 1) { cover = fminf(cover, (float)(cz + kk + 1) - fz); any = true; }
      if (!any) break;
      cover -= kCellMargin;
      if (cover > 0.f && cover * cover * hs2 > bound()) break;
    }
    const int z0 = max(cz - sh, 0), z1 = min(cz + sh, g.nz - 1);
    const int y0 = max(cy - sh, 0), y1 = min(cy + sh, g.ny - 1);
    row_budget -= (z1 - z0 + 1) * (y1 - y0 + 1);
    if (row_budget < 0) {
      reset();
      far_sweep(g, qx, qy, qz, k_needed, bound, scan);
      return;
    }
    const int xl = cx - sh, xr = cx + sh;
    const int x0 = max(xl, 0), x1 = min(xr, g.nx - 1);
    for (int rz = z0; rz <= z1; ++rz) {
      const float gz = slab_gap(fz, cz, rz);
      if (gz * gz * hs2 > bound()) continue;
      const bool zshell = (rz - cz == sh) || (cz - rz == sh);
      for (int ry = y0; ry <= y1; ++ry) {
        const float gy = slab_gap(fy, cy, ry);
        const float gyz2 = gy * gy + gz * gz;
        if (gyz2 * hs2 > bound()) continue;
        const uint32_t base = ((uint32_t)rz * (uint32_t)g.ny + (uint32_t)ry) * (uint32_t)g.nx;
        if (zshell || (ry - cy == sh) || (cy - ry == sh)) {
          if (x0 <= x1) scan(__ldg(g.cell_start + base + x0), __ldg(g.cell_start + base + x1 + 1));
        } else {
          if (xl >= 0 && xl < g.nx) scan(__ldg(g.cell_start + base + xl), __ldg(g.cell_start + base + xl + 1));
          if (sh > 0 && xr >= 0 && xr < g.nx)
            scan(__ldg(g.cell_start + base + xr), __ldg(g.cell_start + base + xr + 1));
        }
      }
    }
  }
}

}  // namespace cb
