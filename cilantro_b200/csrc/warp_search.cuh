// Warp-cooperative exact nearest neighbour over the grid (product code, sm_90a).
//
// Why: in the per-lane search (nn_search.cuh) each of the 10 "residual" regions around a query — the
// two x-neighbour cells and the 8 neighbour rows of shells 0-1 — is needed by only ~5-15 % of the
// lanes once the own cell has been scanned (the match is usually there), but a warp executes a
// region's scan loop if ANY lane needs it, so most of the issued instructions ran at low lane utilisation.
//
// Here the warp pools that work:
//   phase A (per lane)   own-cell scan; decide which of the 10 regions can still hold a closer point;
//                        push one work item (first cell, #cells, lane) per such region into a
//                        warp-private shared-memory queue (ballot + popc, no atomics);
//   phase B (pooled)     lane k takes item k, k+32, ...: every lane is busy scanning a region for SOME
//                        query of the warp; results merge with a 64-bit shared-memory atomicMin on
//                        (d2 bits << 32 | position);
//   phase C (per lane)   read back the merged best, run the termination test of nn_search.cuh; the
//                        rare lanes that are outside the grid, need shell >= 2, or saw a bit-equal
//                        distance (exact-tie rule) fall back to the per-lane exact search.
// Results are identical to grid_nearest() — same candidates, same bounds, same tie rule — which the
// parity tests check bit for bit.
#pragma once
#include "nn_search.cuh"

namespace cb {

constexpr int kWarpItemsMax = 320;  // 10 regions x 32 lanes: the queue can never overflow

struct WarpSearchSmem {
  float4 q[32];                    // query position (x, y, z, unused)
  unsigned long long key[32];      // merged best: d2 bits << 32 | sorted position (0xffffffff = none)
  uint2 item[kWarpItemsMax];       // .x = first cell index, .y = (#cells << 8) | lane
  unsigned int tie_mask;           // lanes that saw a bit-equal distance
  unsigned int pad;
};

__device__ __forceinline__ unsigned long long pack_key(float d2, unsigned int pos) {
  return ((unsigned long long)__float_as_uint(d2) << 32) | (unsigned long long)pos;
}

// All 32 lanes of the warp must call this (inactive lanes pass active = false).
// warm_pos >= 0: sorted position of a point known to be close (the query's match in the previous ICP
// iteration). Its exact distance under the current transform seeds the running best, so most of the 10
// residual regions are pruned before they are queued; the result is unchanged (the seed is a real candidate
// with its exact d2, and a bit-equal distance elsewhere still raises the tie flag).
__device__ __forceinline__ Best warp_grid_nearest(const GridView& g, WarpSearchSmem& sm, bool active, float qx, float qy,
                                                  float qz, float max_d2, int warm_pos = -1) {
  const unsigned int lane = threadIdx.x & 31;
  const unsigned int lt_mask = (1u << lane) - 1u;
  Best best;
  best.d2 = max_d2;
  best.idx = -1;
  best.pos = -1;
  best.tie = false;

  const float fx = cell_coord(qx, g.ox, g.inv_h), fy = cell_coord(qy, g.oy, g.inv_h), fz = cell_coord(qz, g.oz, g.inv_h);
  const int cx = (int)floorf(fx), cy = (int)floorf(fy), cz = (int)floorf(fz);
  const float hs2 = g.hs2;
  const bool inside = active && g.n > 0 && cx >= 0 && cx < g.nx && cy >= 0 && cy < g.ny && cz >= 0 && cz < g.nz;
  bool slow = active && g.n > 0 && !inside;  // outside the grid: per-lane exact search at the end

  if (inside && warm_pos >= 0) {
    const float4 p = __ldg(g.pts + warm_pos);
    const float dx = __fsub_rn(qx, p.x), dy = __fsub_rn(qy, p.y), dz = __fsub_rn(qz, p.z);
    float r = __fmul_rn(dx, dx);
    r = __fadd_rn(r, __fmul_rn(dy, dy));
    r = __fadd_rn(r, __fmul_rn(dz, dz));
    if (r < max_d2) {
      best.d2 = r;
      best.pos = warm_pos;
    }
  }
  if (lane == 0) sm.tie_mask = 0u;
  sm.q[lane] = make_float4(qx, qy, qz, 0.f);
  sm.key[lane] = pack_key(max_d2, 0xffffffffu);
  __syncwarp();

  // ---- phase A: own cell + work items --------------------------------------------------------------
  unsigned int count = 0;  // warp-uniform number of queued items
  {
    const uint32_t cbase = inside ? ((uint32_t)cz * (uint32_t)g.ny + (uint32_t)cy) * (uint32_t)g.nx : 0u;
    uint32_t s1 = 0, s2 = 0;
    if (inside) {
      s1 = __ldg(g.cell_start + cbase + cx);
      s2 = __ldg(g.cell_start + cbase + cx + 1);
    }
    if (inside) scan_range<false>(g.pts, s1, s2, qx, qy, qz, best, best.pos);
    // lower bounds (cells, margin applied) of the 10 residual regions
    const float gxl = slab_gap(fx, cx, cx - 1), gxr = slab_gap(fx, cx, cx + 1);
    const float gym = slab_gap(fy, cy, cy - 1), gyp = slab_gap(fy, cy, cy + 1);
    const float gzm = slab_gap(fz, cz, cz - 1), gzp = slab_gap(fz, cz, cz + 1);
    const float gy2[3] = {gym * gym, 0.f, gyp * gyp};
    const float gz2[3] = {gzm * gzm, 0.f, gzp * gzp};
    const int xm = max(cx - 1, 0), xp = min(cx + 1, g.nx - 1);
    constexpr int kDy[8] = {-1, 1, 0, 0, -1, 1, -1, 1};
    constexpr int kDz[8] = {0, 0, -1, 1, -1, -1, 1, 1};
#pragma unroll
    for (int t = 0; t < 10; ++t) {
      bool need;
      uint32_t first;
      uint32_t ncells;
      if (t == 0) {  // left x-neighbour
        need = inside && cx > 0 && (gxl * gxl * hs2 <= best.d2);
        first = cbase + (uint32_t)(cx - 1);
        ncells = 1;
      } else if (t == 1) {  // right x-neighbour
        need = inside && cx < g.nx - 1 && (gxr * gxr * hs2 <= best.d2);
        first = cbase + (uint32_t)(cx + 1);
        ncells = 1;
      } else {
        const int ry = cy + kDy[t - 2], rz = cz + kDz[t - 2];
        const bool valid = inside && ry >= 0 && ry < g.ny && rz >= 0 && rz < g.nz;
        need = valid && ((gy2[kDy[t - 2] + 1] + gz2[kDz[t - 2] + 1]) * hs2 <= best.d2);
        first = ((uint32_t)rz * (uint32_t)g.ny + (uint32_t)ry) * (uint32_t)g.nx + (uint32_t)xm;
        ncells = (uint32_t)(xp - xm + 1);
      }
      const unsigned int m = __ballot_sync(0xffffffffu, need);
      if (need) sm.item[count + __popc(m & lt_mask)] = make_uint2(first, (ncells << 8) | lane);
      count += __popc(m);
    }
    if (best.pos >= 0) sm.key[lane] = pack_key(best.d2, (unsigned int)best.pos);
    if (best.tie) atomicOr(&sm.tie_mask, 1u << lane);
  }
  __syncwarp();

  // ---- phase B: pooled scan of the queued regions ----------------------------------------------------
  for (unsigned int k = lane; k < count; k += 32) {
    const uint2 it = sm.item[k];
    const unsigned int ql = it.y & 31u, nc = it.y >> 8;
    const float4 q = sm.q[ql];
    const uint32_t b = __ldg(g.cell_start + it.x), e = __ldg(g.cell_start + it.x + nc);
    Best loc;
    // bound = the owner's best when the item was queued or better (merged so far)
    const unsigned long long cur = sm.key[ql];
    loc.d2 = __uint_as_float((unsigned int)(cur >> 32));
    loc.idx = -1;
    loc.pos = -1;
    loc.tie = false;
    scan_range<false>(g.pts, b, e, q.x, q.y, q.z, loc, (int)(unsigned int)(cur & 0xffffffffull));
    if (loc.pos >= 0) {
      const unsigned long long key = pack_key(loc.d2, (unsigned int)loc.pos);
      const unsigned long long old = atomicMin(&sm.key[ql], key);
      if ((old >> 32) == (key >> 32) && old != key) loc.tie = true;  // bit-equal d2 from another region
    }
    if (loc.tie) atomicOr(&sm.tie_mask, 1u << ql);
  }
  __syncwarp();

  // ---- phase C: merged result, termination, rare exact fallbacks -------------------------------------
  if (inside) {
    const unsigned long long key = sm.key[lane];
    const unsigned int pos = (unsigned int)(key & 0xffffffffull);
    best.d2 = __uint_as_float((unsigned int)(key >> 32));
    best.pos = (pos == 0xffffffffu) ? -1 : (int)pos;
    best.tie = (sm.tie_mask >> lane) & 1u;
    // shells 0-1 are complete: same termination test as grid_nearest (kk = 1)
    float cover = 3.0e38f;
    bool any = false;
    if (cx - 1 > 0) { cover = fminf(cover, fx - (float)(cx - 1)); any = true; }
    if (cx + 1 < g.nx - 1) { cover = fminf(cover, (float)(cx + 2) - fx); any = true; }
    if (cy - 1 > 0) { cover = fminf(cover, fy - (float)(cy - 1)); any = true; }
    if (cy + 1 < g.ny - 1) { cover = fminf(cover, (float)(cy + 2) - fy); any = true; }
    if (cz - 1 > 0) { cover = fminf(cover, fz - (float)(cz - 1)); any = true; }
    if (cz + 1 < g.nz - 1) { cover = fminf(cover, (float)(cz + 2) - fz); any = true; }
    cover -= kCellMargin;
    const bool done = !any || (cover > 0.f && cover * cover * hs2 > best.d2);
    if (!done || best.tie) slow = true;
  }
  if (slow) {
    // rare: outside the grid, shell >= 2 needed, or an exact tie to resolve on the original index
    best = grid_nearest(g, qx, qy, qz, max_d2);
  } else if (best.pos >= 0) {
    best.idx = __float_as_int(__ldg(&g.pts[best.pos].w));
  }
  __syncwarp();  // the shared arrays are reused by the caller's next query batch
  return best;
}

}  // namespace cb
