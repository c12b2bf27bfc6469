// Device-side exact nearest-neighbour search over the uniform grid (product code, sm_90a).
//
// Replaces the nanoflann kd-tree descent the reference runs per query
// (core/kd_tree.hpp:284-291 -> 3rd_party/nanoflann/nanoflann.hpp:1709-1732,1886-1961) with a
// bounded sweep over grid cells. Exactness argument (DESIGN.md "Grid search is exact"):
//   * candidates are visited row by row (a row = all cells sharing (y, z)); a row, a cell or a
//     whole shell is skipped only when a lower bound of the fp32 d2 of every point in it is strictly
//     greater than the best squared distance found so far (a bit-equal d2 may still win on its index);
//   * the lower bounds are computed in cell units from the SAME float expression that assigned
//     reference points to cells (cell_coord below), shrunk by 2^-10 cell and scaled by GridView::hs2
//     (h_safe^2, h_safe = h(1-2^-10), clamped finite: grid_view), which dominates the <= 2^-11-cell
//     rounding uncertainty of that expression for grids of <= 1024 cells per axis;
//   * the search ends when the scanned block's nearest face is farther than the best distance.
//
// Every sweep (this file's 1-NN, grid_sweep.cuh, far_sweep.cuh, warp_search.cuh, warp_search_wide.cuh) takes its
// pieces of that argument from here: the query cell (query_cell), the first shell that holds cells (first_shell),
// the row / cell gaps (slab_gap) and the termination test (open_face_gap).
//
// Arithmetic contract (must match oracle/cilantro_oracle.cpp bit for bit; fp32, RN, no FMA): the query is
// rule::transform_point and every candidate's distance rule::contract_d2 (cache_rule.hpp, also compiled for the host
// test); accept iff d2 < max_d2; exact ties -> lowest original reference index.
#pragma once
#include "cache_rule.hpp"
#include "cb_internal.hpp"

namespace cb {

struct Rigid {
  float r[9];  // row-major rotation
  float t[3];
};

// float[12] row-major [R | t] of the C ABI -> Rigid (nullptr = identity)
inline Rigid rigid_from_t12(const float* T12) {
  Rigid r;
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) r.r[i * 3 + j] = T12 ? T12[i * 4 + j] : (i == j ? 1.f : 0.f);
    r.t[i] = T12 ? T12[i * 4 + 3] : 0.f;
  }
  return r;
}

// The one finiteness rule of the grid: a point with a NaN or Inf coordinate is at no finite distance from anything
// (every d2 it takes part in is NaN or Inf, which fails d2 < bound), so it is never searched, never a candidate and
// left out of the grid's extent. Every finite point is searched, up to +-FLT_MAX.
// The quarter-weighted sum is at most 0.75 FLT_MAX for finite coordinates (no overflow) and Inf or NaN otherwise; one
// chain of adds and one compare, as cheap as the sum of magnitudes it replaces on the per-query paths.
__host__ __device__ __forceinline__ bool finite_point(float x, float y, float z) {
  return 0.25f * fabsf(x) + (0.25f * fabsf(y) + 0.25f * fabsf(z)) < INFINITY;
}

__device__ __forceinline__ float sum3(float a0, float a1, float a2) { return __fadd_rn(a0, __fadd_rn(a1, a2)); }

__device__ __forceinline__ void rotate_rigid(const Rigid& T, float x, float y, float z, float& qx, float& qy,
                                             float& qz) {
  qx = sum3(__fmul_rn(T.r[0], x), __fmul_rn(T.r[1], y), __fmul_rn(T.r[2], z));
  qy = sum3(__fmul_rn(T.r[3], x), __fmul_rn(T.r[4], y), __fmul_rn(T.r[5], z));
  qz = sum3(__fmul_rn(T.r[6], x), __fmul_rn(T.r[7], y), __fmul_rn(T.r[8], z));
}

// Continuous cell coordinate of x along one axis. The ONLY expression that maps a coordinate to a
// cell, for reference points (grid build) and queries alike.
__host__ __device__ __forceinline__ float cell_coord(float x, float o, float inv_h) {
#ifdef __CUDA_ARCH__
  float f = __fmul_rn(__fsub_rn(x, o), inv_h);
#else
  float f = (x - o) * inv_h;
#endif
  f = f < -16777216.f ? -16777216.f : f;
  f = f > 16777216.f ? 16777216.f : f;
  return (f == f) ? f : -16777216.f;  // NaN coordinates land far outside
}

// A query in cell units: continuous coordinate f and cell c = floor(f) per axis.
struct QueryCell {
  float fx, fy, fz;
  int cx, cy, cz;
};

__device__ __forceinline__ QueryCell query_cell(const GridView& g, float qx, float qy, float qz) {
  QueryCell c;
  c.fx = cell_coord(qx, g.ox, g.inv_h);
  c.fy = cell_coord(qy, g.oy, g.inv_h);
  c.fz = cell_coord(qz, g.oz, g.inv_h);
  c.cx = (int)floorf(c.fx);
  c.cy = (int)floorf(c.fy);
  c.cz = (int)floorf(c.fz);
  return c;
}

// first Chebyshev shell around the query cell that can contain grid cells at all (0 = the cell is inside the grid)
__device__ __forceinline__ int first_shell(const GridView& g, const QueryCell& c) {
  int k0 = 0;
  k0 = max(k0, c.cx < 0 ? -c.cx : (c.cx > g.nx - 1 ? c.cx - (g.nx - 1) : 0));
  k0 = max(k0, c.cy < 0 ? -c.cy : (c.cy > g.ny - 1 ? c.cy - (g.ny - 1) : 0));
  k0 = max(k0, c.cz < 0 ? -c.cz : (c.cz > g.nz - 1 ? c.cz - (g.nz - 1) : 0));
  return k0;
}

struct Best {
  float d2;
  int idx;   // original reference index, -1 = none
  int pos;   // position in the cell-sorted array
  bool tie;  // fast pass only: some candidate had d2 bit-equal to the running best
};

__device__ __forceinline__ Best no_best(float max_d2) { return Best{max_d2, -1, -1, false}; }

constexpr float kCellMargin = 0.0009765625f;  // 2^-10 cell

__constant__ signed char kRowDy[9] = {0, -1, 1, 0, 0, -1, 1, -1, 1};
__constant__ signed char kRowDz[9] = {0, 0, 0, -1, 1, -1, -1, 1, 1};

// The candidate loop of the pooled searches: eval(d2, j) for every cell-sorted point j of [b, e).
// The scan is a chain of load -> use steps, and the warps mostly wait on those loads (long scoreboard). Batches of
// kW candidates put kW loads in flight per wait; slots past the end of the range are predicated off (no padded
// arithmetic — a padded variant doubled the instruction count and was slower).
template <class Eval>
__device__ __forceinline__ void scan_batched(const float4* __restrict__ pts, uint32_t b, uint32_t e, float qx, float qy,
                                             float qz, Eval&& eval) {
  constexpr int kW = 4;
  for (uint32_t j = b; j < e; j += kW) {
    float4 p[kW];
    p[0] = __ldg(pts + j);
#pragma unroll
    for (int u = 1; u < kW; u++)
      if (j + u < e) p[u] = __ldg(pts + j + u);
    eval(rule::contract_d2(qx, qy, qz, p[0].x, p[0].y, p[0].z), j);
#pragma unroll
    for (int u = 1; u < kW; u++)
      if (j + u < e) eval(rule::contract_d2(qx, qy, qz, p[u].x, p[u].y, p[u].z), j + u);
  }
}

// kExact = true resolves exact ties on the original index inside the loop. kExact = false (the fast
// pass) keeps the first strictly smaller candidate and only RECORDS that a bit-equal distance was
// seen; grid_nearest() then repeats the search with kExact = true for that (very rare) query.
// skip_pos (fast pass only): the position of a point that is ALREADY the running best (a warm start from the
// previous ICP iteration, or the merged best of the warp-pooled search) — meeting it again is not a tie.
template <bool kExact>
__device__ __forceinline__ void scan_range(const float4* __restrict__ pts, uint32_t b, uint32_t e, float qx,
                                           float qy, float qz, Best& best, int skip_pos = -1) {
  if (kExact) {
#pragma unroll 2
    for (uint32_t j = b; j < e; ++j) {
      const float4 p = __ldg(pts + j);
      const float r = rule::contract_d2(qx, qy, qz, p.x, p.y, p.z);
      const int pi = __float_as_int(p.w);
      if (r < best.d2 || (r == best.d2 && pi < best.idx)) {
        best.d2 = r;
        best.idx = pi;
        best.pos = (int)j;
      }
    }
  } else {
    scan_batched(pts, b, e, qx, qy, qz, [&](float r, uint32_t j) {
      if (r < best.d2) {
        best.d2 = r;
        best.pos = (int)j;
      } else if (r == best.d2 && (int)j != skip_pos) {
        best.tie = true;
      }
    });
  }
}

// gap (in cells, >= 0, already shrunk by the safety margin) between coordinate f in cell c and the
// slab of cells [r, r+1).
__device__ __forceinline__ float slab_gap(float f, int c, int r) {
  float g = 0.f;
  if (r > c) g = (float)r - f;
  if (r < c) g = f - (float)(r + 1);
  g -= kCellMargin;
  return g > 0.f ? g : 0.f;
}

// The termination test of every shell sweep. Returns false when the scanned block [c-kk, c+kk] already covers the
// whole grid; otherwise gap receives the distance (cells, shrunk by the margin, may be <= 0) from the query to the
// block's nearest face that still has grid cells beyond it. Every point not yet scanned lies beyond such a face, so
// once gap > 0 and gap^2 hs2 > bound, none of them can pass d2 < bound or tie with it.
__device__ __forceinline__ bool open_face_gap(const GridView& g, const QueryCell& c, int kk, float& gap) {
  float cover = 3.0e38f;
  bool any = false;
  if (c.cx - kk > 0) { cover = fminf(cover, c.fx - (float)(c.cx - kk)); any = true; }
  if (c.cx + kk < g.nx - 1) { cover = fminf(cover, (float)(c.cx + kk + 1) - c.fx); any = true; }
  if (c.cy - kk > 0) { cover = fminf(cover, c.fy - (float)(c.cy - kk)); any = true; }
  if (c.cy + kk < g.ny - 1) { cover = fminf(cover, (float)(c.cy + kk + 1) - c.fy); any = true; }
  if (c.cz - kk > 0) { cover = fminf(cover, c.fz - (float)(c.cz - kk)); any = true; }
  if (c.cz + kk < g.nz - 1) { cover = fminf(cover, (float)(c.cz + kk + 1) - c.fz); any = true; }
  gap = cover - kCellMargin;
  return any;
}

}  // namespace cb

#include "far_sweep.cuh"

namespace cb {

// Exact nearest neighbour of (qx,qy,qz) among the grid's points with d2 < max_d2.
template <bool kExact>
__device__ __forceinline__ Best grid_nearest_impl(const GridView& g, float qx, float qy, float qz, float max_d2) {
  Best best = no_best(max_d2);
  if (g.n == 0) return best;
  if (!finite_point(qx, qy, qz)) return best;

  const QueryCell c = query_cell(g, qx, qy, qz);
  const int cx = c.cx, cy = c.cy, cz = c.cz;
  const float hs2 = g.hs2;
  const int k0 = first_shell(g, c);
  int k = k0;
  if (k0 == 0) {
    // Query cell inside the grid (the common case). Shells 0 and 1: all 20 cell-table entries are
    // requested up front (independent loads, one latency), then the cells are visited from the most
    // to the least promising: own cell, its two x-neighbours, the 4 face rows, the 4 corner rows,
    // each skipped when its lower bound already exceeds the best distance.
    const int xm = max(cx - 1, 0), xp = min(cx + 1, g.nx - 1);
    const uint32_t cbase = ((uint32_t)cz * (uint32_t)g.ny + (uint32_t)cy) * (uint32_t)g.nx;
    const uint32_t s0 = __ldg(g.cell_start + cbase + xm), s1 = __ldg(g.cell_start + cbase + cx);
    const uint32_t s2 = __ldg(g.cell_start + cbase + cx + 1), s3 = __ldg(g.cell_start + cbase + xp + 1);
    constexpr int kDy[8] = {-1, 1, 0, 0, -1, 1, -1, 1};  // 4 face rows, then 4 corner rows
    constexpr int kDz[8] = {0, 0, -1, 1, -1, -1, 1, 1};
    uint32_t rb[8], re[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int ry = cy + kDy[t], rz = cz + kDz[t];
      const bool valid = (ry >= 0) & (ry < g.ny) & (rz >= 0) & (rz < g.nz);
      const uint32_t base = valid ? ((uint32_t)rz * (uint32_t)g.ny + (uint32_t)ry) * (uint32_t)g.nx : cbase;
      const uint32_t b = __ldg(g.cell_start + base + xm), e = __ldg(g.cell_start + base + xp + 1);
      rb[t] = valid ? b : 0u;
      re[t] = valid ? e : 0u;
    }
    scan_range<kExact>(g.pts, s1, s2, qx, qy, qz, best);
    {
      const float gl = slab_gap(c.fx, cx, cx - 1), gr = slab_gap(c.fx, cx, cx + 1);
      if (gl * gl * hs2 <= best.d2) scan_range<kExact>(g.pts, s0, s1, qx, qy, qz, best);
      if (gr * gr * hs2 <= best.d2) scan_range<kExact>(g.pts, s2, s3, qx, qy, qz, best);
    }
    {
      const float gym = slab_gap(c.fy, cy, cy - 1), gyp = slab_gap(c.fy, cy, cy + 1);
      const float gzm = slab_gap(c.fz, cz, cz - 1), gzp = slab_gap(c.fz, cz, cz + 1);
      const float gy2[3] = {gym * gym, 0.f, gyp * gyp};
      const float gz2[3] = {gzm * gzm, 0.f, gzp * gzp};
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const float lb = (gy2[kDy[t] + 1] + gz2[kDz[t] + 1]) * hs2;
        if (lb <= best.d2 && rb[t] < re[t]) scan_range<kExact>(g.pts, rb[t], re[t], qx, qy, qz, best);
      }
    }
    k = 2;
  } else if (k0 == 1) {
    // Shells 0 and 1 together: 9 rows of up to 3 contiguous cells. Centre row first so that the
    // bound is tight before the 8 neighbour rows are tested for pruning.
    const int x0 = max(cx - 1, 0), x1 = min(cx + 1, g.nx - 1);
    if (x0 <= x1) {
#pragma unroll 1
      for (int t = 0; t < 9; ++t) {
        // visiting order: (0,0), then the 4 face rows, then the 4 corner rows
        const int ry = cy + kRowDy[t], rz = cz + kRowDz[t];
        if (ry < 0 || ry >= g.ny || rz < 0 || rz >= g.nz) continue;
        const float gy = slab_gap(c.fy, cy, ry), gz = slab_gap(c.fz, cz, rz);
        if ((gy * gy + gz * gz) * hs2 > best.d2) continue;
        const uint32_t base = ((uint32_t)rz * (uint32_t)g.ny + (uint32_t)ry) * (uint32_t)g.nx;
        const uint32_t b = __ldg(g.cell_start + base + x0), e = __ldg(g.cell_start + base + x1 + 1);
        scan_range<kExact>(g.pts, b, e, qx, qy, qz, best);
      }
    }
    k = 2;
  }

  // Shells < k are done. Same walk as grid_sweep (grid_sweep.cuh), plus an x-gap prune of the two end cells of
  // inner rows.
  int row_budget = kFarRowBudget;
#pragma unroll 1
  for (;; ++k) {
    {
      float cover;
      if (!open_face_gap(g, c, k - 1, cover)) break;  // the whole grid has been scanned
      if (cover > 0.f && cover * cover * hs2 > best.d2) break;
    }
    // Shell k: rows with max(|dy|,|dz|) == k take the full x-extent, inner rows only the two end cells.
    const int z0 = max(cz - k, 0), z1 = min(cz + k, g.nz - 1);
    const int y0 = max(cy - k, 0), y1 = min(cy + k, g.ny - 1);
    row_budget -= (z1 - z0 + 1) * (y1 - y0 + 1);
    if (row_budget < 0) {
      // too much (mostly empty) space crossed shell by shell: restart on the list of non-empty blocks
      best = no_best(max_d2);
      far_sweep(
          g, qx, qy, qz, 1u, [&]() { return best.d2; },
          [&](uint32_t b, uint32_t e) { scan_range<kExact>(g.pts, b, e, qx, qy, qz, best); });
      break;
    }
    const int xl = cx - k, xr = cx + k;
    const int x0 = max(xl, 0), x1 = min(xr, g.nx - 1);
    for (int rz = z0; rz <= z1; ++rz) {
      const float gz = slab_gap(c.fz, cz, rz);
      const float gz2 = gz * gz;
      if (gz2 * hs2 > best.d2) continue;
      const bool zshell = (rz - cz == k) || (cz - rz == k);
      for (int ry = y0; ry <= y1; ++ry) {
        const float gy = slab_gap(c.fy, cy, ry);
        const float gyz2 = gy * gy + gz2;
        if (gyz2 * hs2 > best.d2) continue;
        const uint32_t base = ((uint32_t)rz * (uint32_t)g.ny + (uint32_t)ry) * (uint32_t)g.nx;
        if (zshell || (ry - cy == k) || (cy - ry == k)) {
          if (x0 <= x1) {
            const uint32_t b = __ldg(g.cell_start + base + x0), e = __ldg(g.cell_start + base + x1 + 1);
            scan_range<kExact>(g.pts, b, e, qx, qy, qz, best);
          }
        } else {
          if (xl >= 0 && xl < g.nx) {
            const float gx = slab_gap(c.fx, cx, xl);
            if ((gx * gx + gyz2) * hs2 <= best.d2) {
              const uint32_t b = __ldg(g.cell_start + base + xl), e = __ldg(g.cell_start + base + xl + 1);
              scan_range<kExact>(g.pts, b, e, qx, qy, qz, best);
            }
          }
          if (xr >= 0 && xr < g.nx) {
            const float gx = slab_gap(c.fx, cx, xr);
            if ((gx * gx + gyz2) * hs2 <= best.d2) {
              const uint32_t b = __ldg(g.cell_start + base + xr), e = __ldg(g.cell_start + base + xr + 1);
              scan_range<kExact>(g.pts, b, e, qx, qy, qz, best);
            }
          }
        }
      }
    }
  }
  if (!kExact && best.pos >= 0) best.idx = __float_as_int(__ldg(&g.pts[best.pos].w));
  return best;
}

__device__ __forceinline__ Best grid_nearest(const GridView& g, float qx, float qy, float qz, float max_d2) {
  Best best = grid_nearest_impl<false>(g, qx, qy, qz, max_d2);
  if (best.tie) best = grid_nearest_impl<true>(g, qx, qy, qz, max_d2);
  return best;
}

}  // namespace cb
