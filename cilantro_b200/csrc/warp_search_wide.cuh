// Warp-cooperative exact nearest neighbour WITH an exclusion bound (product code, sm_90a).
//
// Same search as warp_grid_nearest() (warp_search.cuh) — same candidates' arithmetic, same conservative
// region bounds, same tie rule, hence the same (index, d2) bit for bit — plus one more output:
//
//   D2 = a lower bound of the squared distance from the query to EVERY reference point other than the
//        returned best ("the second-nearest point is at least sqrt(D2) away").
//
// The device-resident ICP loop (icp_loop.cu) caches (best, sqrt(D2)) per query: in the next iteration the
// query has moved by delta = |T' s - T s|, so every other point is still at least sqrt(D2) - delta away
// (triangle inequality), and if the cached match's new distance is below that, it is provably still the
// exact nearest neighbour — no grid access at all. To make D2 useful the search is WIDENED: after the own
// cell, a region is scanned iff its lower bound is below (sqrt(best) + slack)^2 instead of best, the two
// smallest distances are tracked instead of one, and D2 = min(second smallest scanned, the widened bound,
// the squared distance to the boundary of the scanned 3x3x3 block).
// The shared-memory arrays and item decode (warp_search.cuh), the 4-wide candidate loop and the termination test
// (nn_search.cuh) are the narrow search's; with kGroup > 1 lanes per region, phase B has its own interleaved loop. Phase A keeps its own copy of the region enumeration (compared against
// wide2 instead of the best distance): calling queue_regions() here costs the <3,*> search kernels 4-12 B of spills.
#pragma once
#include "warp_search.cuh"

namespace cb {

struct WideSearchSmem : WarpQueue {
  unsigned int sec[32];  // merged second-smallest d2 (float bits; non-negative floats order like uints)
};
// The cached pass of the ICP loop keeps 8 of these per block and is 176 B short of losing a resident block per SM.
static_assert(sizeof(WideSearchSmem) <= 3456, "WideSearchSmem must not grow");

struct WideBest {
  float d2;   // squared distance of the nearest point with d2 < max_d2 (else max_d2)
  int idx;    // its original index, -1 = none
  int pos;    // its position in the cell-sorted array, -1 = none
  float D2;   // every OTHER reference point has true squared distance >= D2 (0 = unknown)
};

// two smallest of the candidates seen so far: (b1, p1) and b2; a candidate bit-equal to b1 lands in b2
__device__ __forceinline__ void two_smallest(float r, int j, float& b1, int& p1, float& b2) {
  if (r < b1) {
    b2 = b1;
    b1 = r;
    p1 = j;
  } else {
    b2 = fminf(b2, r);
  }
}

// scans [b, e) tracking the two smallest distances; position `skip` (already accounted for) is ignored
__device__ __forceinline__ void scan_range_two(const float4* __restrict__ pts, uint32_t b, uint32_t e, float qx, float qy,
                                               float qz, float& b1, int& p1, float& b2, int skip) {
  scan_batched(pts, b, e, qx, qy, qz, [&](float r, uint32_t j) {
    if ((int)j != skip) two_smallest(r, (int)j, b1, p1, b2);
  });
}

// A region's two smallest distances (l1 at sorted position lp >= 0, l2) into the owner's merged (key, sec).
__device__ __forceinline__ void merge_region(WideSearchSmem& sm, unsigned int owner, float l1, int lp, float l2,
                                             float max_d2) {
  constexpr float kInf = 3.402823466e+38f;
  float loser = l1;  // what this region contributes to "second smallest" besides l2
  if (l1 < max_d2) {
    const unsigned long long key = pack_key(l1, (unsigned int)lp);
    const unsigned long long old = atomicMin(&sm.key[owner], key);
    const float od2 = __uint_as_float((unsigned int)(old >> 32));
    // the loser of (previous best, this region's best) is a second-best candidate; the initial "none"
    // sentinel is not a point
    loser = ((unsigned int)(old & 0xffffffffull) == 0xffffffffu) ? kInf : fmaxf(od2, l1);
  }
  atomicMin(&sm.sec[owner], __float_as_uint(fminf(l2, loser)));
}

// All 32 lanes of the warp must call this (inactive lanes pass active = false).
// kGroup: lanes per queued region in the pooled scan of phase B (1, 2, 4, ... 32).
// warm_pos >= 0: sorted position of a point known to be close (the cached match); slack >= 0: widening of the
// search radius beyond the nearest distance, in the units of the coordinates.
template <unsigned int kGroup>
__device__ __forceinline__ WideBest warp_grid_nearest_wide(const GridView& g, WideSearchSmem& sm, bool active, float qx,
                                                           float qy, float qz, float max_d2, int warm_pos, float slack) {
  const unsigned int lane = threadIdx.x & 31;
  const unsigned int lt_mask = (1u << lane) - 1u;
  constexpr float kInf = 3.402823466e+38f;
  WideBest out;
  out.d2 = max_d2;
  out.idx = -1;
  out.pos = -1;
  out.D2 = 0.f;

  const QueryCell c = query_cell(g, qx, qy, qz);
  const bool inside = active && g.n > 0 && c.cx >= 0 && c.cx < g.nx && c.cy >= 0 && c.cy < g.ny && c.cz >= 0 && c.cz < g.nz;
  bool slow = active && g.n > 0 && !inside;  // outside the grid: per-lane exact search at the end

  float b1 = kInf, b2 = kInf;  // two smallest distances over ALL scanned candidates (regardless of max_d2)
  int p1 = -1;
  if (inside && warm_pos >= 0) {
    const float4 p = __ldg(g.pts + warm_pos);
    b1 = rule::contract_d2(qx, qy, qz, p.x, p.y, p.z);
    p1 = warm_pos;
  }
  sm.q[lane] = make_float4(qx, qy, qz, 0.f);
  __syncwarp();

  // ---- phase A: own cell + work items --------------------------------------------------------------
  unsigned int count = 0;  // warp-uniform number of queued items
  float wide2 = 0.f;       // regions with a lower bound > wide2 are not scanned
  {
    const uint32_t cbase = inside ? ((uint32_t)c.cz * (uint32_t)g.ny + (uint32_t)c.cy) * (uint32_t)g.nx : 0u;
    uint32_t s1 = 0, s2 = 0;
    if (inside) {
      s1 = __ldg(g.cell_start + cbase + c.cx);
      s2 = __ldg(g.cell_start + cbase + c.cx + 1);
      scan_range_two(g.pts, s1, s2, qx, qy, qz, b1, p1, b2, warm_pos);
    }
    {
      // widened bound: (sqrt(min(b1, max_d2)) + slack)^2, rounded up
      const float w = __fadd_ru(__fsqrt_ru(fminf(b1, max_d2)), slack);
      wide2 = __fmul_ru(w, w);
    }
    const float gxl = slab_gap(c.fx, c.cx, c.cx - 1), gxr = slab_gap(c.fx, c.cx, c.cx + 1);
    const float gym = slab_gap(c.fy, c.cy, c.cy - 1), gyp = slab_gap(c.fy, c.cy, c.cy + 1);
    const float gzm = slab_gap(c.fz, c.cz, c.cz - 1), gzp = slab_gap(c.fz, c.cz, c.cz + 1);
    const float gy2[3] = {gym * gym, 0.f, gyp * gyp};
    const float gz2[3] = {gzm * gzm, 0.f, gzp * gzp};
    const int xm = max(c.cx - 1, 0), xp = min(c.cx + 1, g.nx - 1);
    constexpr int kDy[8] = {-1, 1, 0, 0, -1, 1, -1, 1};
    constexpr int kDz[8] = {0, 0, -1, 1, -1, -1, 1, 1};
    // (Tried: a 10-bit need mask per lane, ONE warp scan and lane-major item order instead of a ballot per region -
    // fewer instructions but slower: region-major order
    // makes neighbouring lanes of the pooled scan read neighbouring rows of the sorted array.)
#pragma unroll
    for (int t = 0; t < 10; ++t) {
      bool need;
      uint32_t first;
      uint32_t ncells;
      if (t == 0) {  // left x-neighbour
        need = inside && c.cx > 0 && (gxl * gxl * g.hs2 <= wide2);
        first = cbase + (uint32_t)(c.cx - 1);
        ncells = 1;
      } else if (t == 1) {  // right x-neighbour
        need = inside && c.cx < g.nx - 1 && (gxr * gxr * g.hs2 <= wide2);
        first = cbase + (uint32_t)(c.cx + 1);
        ncells = 1;
      } else {
        const int ry = c.cy + kDy[t - 2], rz = c.cz + kDz[t - 2];
        const bool valid = inside && ry >= 0 && ry < g.ny && rz >= 0 && rz < g.nz;
        need = valid && ((gy2[kDy[t - 2] + 1] + gz2[kDz[t - 2] + 1]) * g.hs2 <= wide2);
        first = ((uint32_t)rz * (uint32_t)g.ny + (uint32_t)ry) * (uint32_t)g.nx + (uint32_t)xm;
        ncells = (uint32_t)(xp - xm + 1);
      }
      const unsigned int m = __ballot_sync(0xffffffffu, need);
      if (need) sm.item[count + __popc(m & lt_mask)] = make_uint2(first, (ncells << 8) | lane);
      count += __popc(m);
    }
    // a candidate at or beyond the radius can never be the match: it only bounds the others
    if (b1 < max_d2) {
      sm.key[lane] = pack_key(b1, (unsigned int)p1);
      sm.sec[lane] = __float_as_uint(b2);
    } else {
      sm.key[lane] = pack_key(max_d2, 0xffffffffu);
      sm.sec[lane] = __float_as_uint(b1);  // b1 <= b2
    }
  }
  __syncwarp();

  // ---- phase B: pooled scan of the queued regions ----------------------------------------------------
  static_assert(kGroup >= 1 && kGroup <= 32 && (kGroup & (kGroup - 1)) == 0, "lanes per region: a power of two");
  if constexpr (kGroup == 1) {
    for (unsigned int k = lane; k < count; k += 32) {
      const QueueItem it = queue_item(g, sm, k);
      if (it.b >= it.e) continue;
      const unsigned long long cur = sm.key[it.lane];
      float l1 = kInf, l2 = kInf;
      int lp = -1;
      // the only point that can be met twice is the warm seed, and only while it is the running best
      scan_range_two(g.pts, it.b, it.e, it.q.x, it.q.y, it.q.z, l1, lp, l2, (int)(unsigned int)(cur & 0xffffffffull));
      if (lp < 0) continue;
      merge_region(sm, it.lane, l1, lp, l2, max_d2);
    }
  } else {
    // kGroup neighbouring lanes share an item and read its points interleaved (two per lane per step). The group's
    // two smallest distances are combined with shuffles, and its first lane merges them into the owner's (key, sec).
    // The result is the same: the two smallest of the same candidates, the warm seed skipped on the same rule.
    const unsigned int sub = lane & (kGroup - 1u);
    for (unsigned int k0 = 0; k0 < count; k0 += 32u / kGroup) {
      const unsigned int k = k0 + lane / kGroup;
      float l1 = kInf, l2 = kInf;
      int lp = -1;
      unsigned int owner = 0;
      if (k < count) {
        const QueueItem it = queue_item(g, sm, k);
        owner = it.lane;
        // the only point that can be met twice is the warm seed, and only while it is the running best
        const int skip = (int)(unsigned int)(sm.key[it.lane] & 0xffffffffull);
        for (uint32_t j = it.b + sub; j < it.e; j += 2u * kGroup) {
          const float4 p0 = __ldg(g.pts + j);
          const bool has1 = j + kGroup < it.e;
          float4 p1 = p0;
          if (has1) p1 = __ldg(g.pts + j + kGroup);
          const float r0 = rule::contract_d2(it.q.x, it.q.y, it.q.z, p0.x, p0.y, p0.z);
          if ((int)j != skip) two_smallest(r0, (int)j, l1, lp, l2);
          if (has1) {
            const float r1 = rule::contract_d2(it.q.x, it.q.y, it.q.z, p1.x, p1.y, p1.z);
            if ((int)(j + kGroup) != skip) two_smallest(r1, (int)(j + kGroup), l1, lp, l2);
          }
        }
      }
      // two smallest of the group: the larger of the two minima is a second-smallest candidate (a bit-equal pair
      // leaves l2 == l1, which phase C reads as a tie)
#pragma unroll
      for (unsigned int m = 1; m < kGroup; m <<= 1) {
        const float o1 = __shfl_xor_sync(0xffffffffu, l1, m), o2 = __shfl_xor_sync(0xffffffffu, l2, m);
        const int op = __shfl_xor_sync(0xffffffffu, lp, m);
        l2 = fminf(fmaxf(l1, o1), fminf(l2, o2));
        if (o1 < l1 || (o1 == l1 && op > lp)) {
          l1 = o1;
          lp = op;
        }
      }
      if (sub == 0 && lp >= 0) merge_region(sm, owner, l1, lp, l2, max_d2);
    }
  }
  __syncwarp();

  // ---- phase C: merged result, termination, exclusion bound, rare exact fallbacks -----------------------
  if (inside) {
    const unsigned long long key = sm.key[lane];
    const unsigned int pos = (unsigned int)(key & 0xffffffffull);
    out.d2 = __uint_as_float((unsigned int)(key >> 32));
    out.pos = (pos == 0xffffffffu) ? -1 : (int)pos;
    const float sec = __uint_as_float(sm.sec[lane]);
    // shells 0-1 are complete: squared distance to the nearest face with grid cells beyond it (kInf: none)
    float cover;
    const bool any = open_face_gap(g, c, 1, cover);
    const float cover2 = (!any) ? kInf : (cover > 0.f ? cover * cover * g.hs2 : 0.f);
    const bool done = cover2 > out.d2;
    const bool tie = out.pos >= 0 && sec == out.d2;  // a second point at a bit-equal distance: index rule
    if (!done || tie) slow = true;
    out.D2 = fminf(fminf(sec, wide2), cover2);
  }
  if (slow) {
    // rare: outside the grid, shell >= 2 needed, or an exact tie to resolve on the original index.
    // No exclusion bound: the next iteration searches this query again.
    const Best bst = grid_nearest(g, qx, qy, qz, max_d2);
    out.d2 = bst.d2;
    out.idx = bst.idx;
    out.pos = bst.pos;
    out.D2 = 0.f;
  } else if (out.pos >= 0) {
    out.idx = __float_as_int(__ldg(&g.pts[out.pos].w));
  }
  __syncwarp();  // the shared arrays are reused by the caller's next query batch
  return out;
}

}  // namespace cb
