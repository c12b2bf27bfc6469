// Warp-cooperative exact nearest neighbour over the grid (product code, sm_90a).
//
// Why: in the per-lane search (nn_search.cuh) each of the 10 "residual" regions around a query — the
// two x-neighbour cells and the 8 neighbour rows of shells 0-1 — is needed by only ~5-15 % of the
// lanes once the own cell has been scanned (the match is usually there), but a warp executes a
// region's scan loop if ANY lane needs it, so most of the issued instructions ran at low lane utilisation.
//
// Here the warp pools that work:
//   phase A (per lane)   own-cell scan; queue_regions() pushes one work item (first cell, #cells, lane) per
//                        region that can still hold a closer point into a warp-private shared-memory queue
//                        (ballot + popc, no atomics);
//   phase B (pooled)     lane k takes item k, k+32, ... (queue_item()): every lane is busy scanning a region for
//                        SOME query of the warp; results merge with a 64-bit shared-memory atomicMin on
//                        (d2 bits << 32 | position);
//   phase C (per lane)   read back the merged best, run the termination test of nn_search.cuh (open_face_gap);
//                        the rare lanes that are outside the grid, need shell >= 2, or saw a bit-equal
//                        distance (exact-tie rule) fall back to the per-lane exact search.
// The shared-memory arrays, the item decode and the 4-wide candidate loop (scan_batched) are shared with the widened
// search of warp_search_wide.cuh. Results are identical to grid_nearest() — same candidates, same bounds, same tie rule —
// which the parity tests check bit for bit.
#pragma once
#include "nn_search.cuh"

namespace cb {

constexpr int kWarpItemsMax = 320;  // 10 regions x 32 lanes: the queue can never overflow

// Per-warp shared memory of the pooled searches.
struct WarpQueue {
  float4 q[32];                    // query position (x, y, z, unused)
  unsigned long long key[32];      // merged best: d2 bits << 32 | sorted position (0xffffffff = none)
  uint2 item[kWarpItemsMax];       // .x = first cell index, .y = (#cells << 8) | lane
};

struct WarpSearchSmem : WarpQueue {
  unsigned int tie_mask;           // lanes that saw a bit-equal distance
  unsigned int pad;
};

__device__ __forceinline__ unsigned long long pack_key(float d2, unsigned int pos) {
  return ((unsigned long long)__float_as_uint(d2) << 32) | (unsigned long long)pos;
}

// Phase A after the own cell: queue every residual region of shells 0-1 whose lower bound is <= bound — the left
// and right x-neighbour cells, the 4 face rows, the 4 corner rows — and return the warp-uniform item count. Lanes
// with !inside queue nothing. All 32 lanes must call this.
// The items are region-major: neighbouring lanes of the pooled scan then read neighbouring rows of the sorted array.
// (Tried: a 10-bit need mask per lane, ONE warp scan and lane-major item order instead of a ballot per region —
// fewer instructions but slower.)
__device__ __forceinline__ unsigned int queue_regions(const GridView& g, WarpQueue& sm, const QueryCell& c, bool inside,
                                                      float bound) {
  const unsigned int lane = threadIdx.x & 31;
  const unsigned int lt_mask = (1u << lane) - 1u;
  const float hs2 = g.hs2;
  const uint32_t cbase = inside ? ((uint32_t)c.cz * (uint32_t)g.ny + (uint32_t)c.cy) * (uint32_t)g.nx : 0u;
  // lower bounds (cells, margin applied) of the 10 residual regions
  const float gxl = slab_gap(c.fx, c.cx, c.cx - 1), gxr = slab_gap(c.fx, c.cx, c.cx + 1);
  const float gym = slab_gap(c.fy, c.cy, c.cy - 1), gyp = slab_gap(c.fy, c.cy, c.cy + 1);
  const float gzm = slab_gap(c.fz, c.cz, c.cz - 1), gzp = slab_gap(c.fz, c.cz, c.cz + 1);
  const float gy2[3] = {gym * gym, 0.f, gyp * gyp};
  const float gz2[3] = {gzm * gzm, 0.f, gzp * gzp};
  const int xm = max(c.cx - 1, 0), xp = min(c.cx + 1, g.nx - 1);
  constexpr int kDy[8] = {-1, 1, 0, 0, -1, 1, -1, 1};
  constexpr int kDz[8] = {0, 0, -1, 1, -1, -1, 1, 1};
  unsigned int count = 0;
#pragma unroll
  for (int t = 0; t < 10; ++t) {
    bool need;
    uint32_t first;
    uint32_t ncells;
    if (t == 0) {  // left x-neighbour
      need = inside && c.cx > 0 && (gxl * gxl * hs2 <= bound);
      first = cbase + (uint32_t)(c.cx - 1);
      ncells = 1;
    } else if (t == 1) {  // right x-neighbour
      need = inside && c.cx < g.nx - 1 && (gxr * gxr * hs2 <= bound);
      first = cbase + (uint32_t)(c.cx + 1);
      ncells = 1;
    } else {
      const int ry = c.cy + kDy[t - 2], rz = c.cz + kDz[t - 2];
      const bool valid = inside && ry >= 0 && ry < g.ny && rz >= 0 && rz < g.nz;
      need = valid && ((gy2[kDy[t - 2] + 1] + gz2[kDz[t - 2] + 1]) * hs2 <= bound);
      first = ((uint32_t)rz * (uint32_t)g.ny + (uint32_t)ry) * (uint32_t)g.nx + (uint32_t)xm;
      ncells = (uint32_t)(xp - xm + 1);
    }
    const unsigned int m = __ballot_sync(0xffffffffu, need);
    if (need) sm.item[count + __popc(m & lt_mask)] = make_uint2(first, (ncells << 8) | lane);
    count += __popc(m);
  }
  return count;
}

// Phase B: item k of the queue decoded — the lane that owns it, that lane's query and the sorted range [b, e).
struct QueueItem {
  unsigned int lane;
  float4 q;
  uint32_t b, e;
};

__device__ __forceinline__ QueueItem queue_item(const GridView& g, const WarpQueue& sm, unsigned int k) {
  const uint2 it = sm.item[k];
  QueueItem r;
  r.lane = it.y & 31u;
  r.q = sm.q[r.lane];
  r.b = __ldg(g.cell_start + it.x);
  r.e = __ldg(g.cell_start + it.x + (it.y >> 8));
  return r;
}

// All 32 lanes of the warp must call this (inactive lanes pass active = false).
// warm_pos >= 0: sorted position of a point known to be close (the query's match in the previous ICP
// iteration). Its exact distance under the current transform seeds the running best, so most of the 10
// residual regions are pruned before they are queued; the result is unchanged (the seed is a real candidate
// with its exact d2, and a bit-equal distance elsewhere still raises the tie flag).
__device__ __forceinline__ Best warp_grid_nearest(const GridView& g, WarpSearchSmem& sm, bool active, float qx, float qy,
                                                  float qz, float max_d2, int warm_pos = -1) {
  const unsigned int lane = threadIdx.x & 31;
  Best best = no_best(max_d2);

  const QueryCell c = query_cell(g, qx, qy, qz);
  const bool inside = active && g.n > 0 && c.cx >= 0 && c.cx < g.nx && c.cy >= 0 && c.cy < g.ny && c.cz >= 0 && c.cz < g.nz;
  bool slow = active && g.n > 0 && !inside;  // outside the grid: per-lane exact search at the end

  if (inside && warm_pos >= 0) {
    const float4 p = __ldg(g.pts + warm_pos);
    const float r = rule::contract_d2(qx, qy, qz, p.x, p.y, p.z);
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
  {
    const uint32_t cbase = inside ? ((uint32_t)c.cz * (uint32_t)g.ny + (uint32_t)c.cy) * (uint32_t)g.nx : 0u;
    uint32_t s1 = 0, s2 = 0;
    if (inside) {
      s1 = __ldg(g.cell_start + cbase + c.cx);
      s2 = __ldg(g.cell_start + cbase + c.cx + 1);
    }
    if (inside) scan_range<false>(g.pts, s1, s2, qx, qy, qz, best, best.pos);
  }
  const unsigned int count = queue_regions(g, sm, c, inside, best.d2);
  if (best.pos >= 0) sm.key[lane] = pack_key(best.d2, (unsigned int)best.pos);
  if (best.tie) atomicOr(&sm.tie_mask, 1u << lane);
  __syncwarp();

  // ---- phase B: pooled scan of the queued regions ----------------------------------------------------
  for (unsigned int k = lane; k < count; k += 32) {
    const QueueItem it = queue_item(g, sm, k);
    // bound = the owner's best when the item was queued or better (merged so far)
    const unsigned long long cur = sm.key[it.lane];
    Best loc = no_best(__uint_as_float((unsigned int)(cur >> 32)));
    scan_range<false>(g.pts, it.b, it.e, it.q.x, it.q.y, it.q.z, loc, (int)(unsigned int)(cur & 0xffffffffull));
    if (loc.pos >= 0) {
      const unsigned long long key = pack_key(loc.d2, (unsigned int)loc.pos);
      const unsigned long long old = atomicMin(&sm.key[it.lane], key);
      if ((old >> 32) == (key >> 32) && old != key) loc.tie = true;  // bit-equal d2 from another region
    }
    if (loc.tie) atomicOr(&sm.tie_mask, 1u << it.lane);
  }
  __syncwarp();

  // ---- phase C: merged result, termination, rare exact fallbacks -------------------------------------
  if (inside) {
    const unsigned long long key = sm.key[lane];
    const unsigned int pos = (unsigned int)(key & 0xffffffffull);
    best.d2 = __uint_as_float((unsigned int)(key >> 32));
    best.pos = (pos == 0xffffffffu) ? -1 : (int)pos;
    best.tie = (sm.tie_mask >> lane) & 1u;
    // shells 0-1 are complete: the termination test of the shell walk with kk = 1
    float cover;
    const bool any = open_face_gap(g, c, 1, cover);
    const bool done = !any || (cover > 0.f && cover * cover * g.hs2 > best.d2);
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
