// Generic shell sweep over the uniform grid (product code, sm_90a): visits, for one query, every cell
// range that can still hold a point closer than bound(), in growing Chebyshev shells around the query's
// cell. The query cell, the first shell, the row gaps and the termination test are nn_search.cuh's (2^-10 cell
// margin, hs2), as is the far-query restart (far_sweep.cuh). bound() may shrink while scanning (k-best lists) or
// stay constant (radius neighbourhoods).
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
  const QueryCell c = query_cell(g, qx, qy, qz);
  const float hs2 = g.hs2;
  int row_budget = kFarRowBudget;
  for (int sh = first_shell(g, c);; ++sh) {
    if (sh > 0) {
      // a point beyond the face has a d2 strictly greater than the bound, so it cannot enter even on a tie
      float cover;
      if (!open_face_gap(g, c, sh - 1, cover)) break;
      if (cover > 0.f && cover * cover * hs2 > bound()) break;
    }
    const int z0 = max(c.cz - sh, 0), z1 = min(c.cz + sh, g.nz - 1);
    const int y0 = max(c.cy - sh, 0), y1 = min(c.cy + sh, g.ny - 1);
    row_budget -= (z1 - z0 + 1) * (y1 - y0 + 1);
    if (row_budget < 0) {
      reset();
      far_sweep(g, qx, qy, qz, k_needed, bound, scan);
      return;
    }
    const int xl = c.cx - sh, xr = c.cx + sh;
    const int x0 = max(xl, 0), x1 = min(xr, g.nx - 1);
    for (int rz = z0; rz <= z1; ++rz) {
      const float gz = slab_gap(c.fz, c.cz, rz);
      if (gz * gz * hs2 > bound()) continue;
      const bool zshell = (rz - c.cz == sh) || (c.cz - rz == sh);
      for (int ry = y0; ry <= y1; ++ry) {
        const float gy = slab_gap(c.fy, c.cy, ry);
        const float gyz2 = gy * gy + gz * gz;
        if (gyz2 * hs2 > bound()) continue;
        const uint32_t base = ((uint32_t)rz * (uint32_t)g.ny + (uint32_t)ry) * (uint32_t)g.nx;
        if (zshell || (ry - c.cy == sh) || (c.cy - ry == sh)) {
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
