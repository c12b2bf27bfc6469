// Radius neighbourhood lists over the grid (product code, sm_90a), shared by cb_radius_search (knn_k.cu) and
// mean-shift (mean_shift.cu).
// KDTree::radiusSearch batched (core/kd_tree.hpp:250-278): every ref point with d2 < radius2, ascending
// distance (RadiusSearchResultAdaptor + std::sort by value, :111-141, :254). Three kernels over the same
// sweep: count per query -> exclusive scan -> fill, then one thread per query heap-sorts its segment on
// (d2, original index) — a total order, so the result does not depend on the visiting order (the reference
// leaves the order of equal distances to std::sort).
// Query i is qry[i] with .w = __int_as_float(its slot): counts[slot] (count pass) and offsets[slot] (fill pass).
#pragma once
#include "cb_internal.hpp"
#include "grid_sweep.cuh"

namespace {

constexpr int kRadiusBlock = 128;  // block size of radius_kernel launches

template <bool kFill>
__global__ void __launch_bounds__(kRadiusBlock) radius_kernel(const cb::GridView g, const float4* __restrict__ qry,
                                                              uint32_t nq, const cb::Rigid T, float r2,
                                                              uint32_t* __restrict__ counts,
                                                              const uint32_t* __restrict__ offsets,
                                                              int* __restrict__ out_idx, float* __restrict__ out_d2) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t qi = blockIdx.x * blockDim.x + threadIdx.x; qi < nq; qi += stride) {
    const float4 s = __ldg(qry + qi);
    const int oi = __float_as_int(s.w);
    float qx, qy, qz;
    cb::rule::transform_point(T, s.x, s.y, s.z, qx, qy, qz);
    uint32_t n = 0;
    const uint32_t base = kFill ? offsets[oi] : 0u;
    cb::grid_sweep(
        g, qx, qy, qz, [&]() { return r2; },
        [&](uint32_t b, uint32_t e) {
          for (uint32_t j = b; j < e; ++j) {
            const float4 p = __ldg(g.pts + j);
            const float r = cb::rule::contract_d2(qx, qy, qz, p.x, p.y, p.z);
            if (r < r2) {
              if (kFill) {
                out_idx[base + n] = __float_as_int(p.w);
                out_d2[base + n] = r;
              }
              ++n;
            }
          }
        },
        [&]() { n = 0; }, 0u);
    if (!kFill) counts[oi] = n;
  }
}

__device__ __forceinline__ bool nb_less(float da, int ia, float db, int ib) { return da < db || (da == db && ia < ib); }

__global__ void segment_heapsort_kernel(const uint32_t* __restrict__ offsets, uint32_t nq, int* __restrict__ idx,
                                        float* __restrict__ d2) {
  for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += gridDim.x * blockDim.x) {
    const uint32_t b = offsets[q], m = offsets[q + 1] - b;
    if (m < 2) continue;
    int* I = idx + b;
    float* D = d2 + b;
    auto sift = [&](uint32_t root, uint32_t end) {  // max-heap on (d2, idx)
      const float dv = D[root];
      const int iv = I[root];
      for (;;) {
        uint32_t c = 2 * root + 1;
        if (c >= end) break;
        if (c + 1 < end && nb_less(D[c], I[c], D[c + 1], I[c + 1])) ++c;
        if (!nb_less(dv, iv, D[c], I[c])) break;
        D[root] = D[c];
        I[root] = I[c];
        root = c;
      }
      D[root] = dv;
      I[root] = iv;
    };
    for (uint32_t s = m / 2; s-- > 0;) sift(s, m);
    for (uint32_t e = m - 1; e > 0; --e) {
      const float dt = D[0];
      const int it = I[0];
      D[0] = D[e];
      I[0] = I[e];
      D[e] = dt;
      I[e] = it;
      sift(0, e);
    }
  }
}

}  // namespace
