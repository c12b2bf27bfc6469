// Feature-space correspondence search of the rigid ICP (product code, sm_90a).
// Replaces the kd-tree CorrespondenceSearchKDTree<PointNormal / PointColor / PointNormalColorFeaturesAdaptor3f> builds
// over the features (correspondence_search/correspondence_search_kd_tree.hpp:107-229 with
// common_transformable_feature_adaptors.hpp) by the 3-D grid of the points and the distance of feature_rule.hpp.
//
// Layout: the tails (w_n n and / or w_c c, feature_rule.hpp) of a grid's points sit in a companion array in the grid's
// cell order, one float4 per tail (16 B per point with one tail, 32 B with two), next to the float4 xyz copy.
// Walk: grid_sweep.cuh (the shell walk, its gaps and termination test, the far-query restart of far_sweep.cuh) with
// k_needed = 0; every bound it prunes with is a lower bound of the xyz part, hence of the feature distance
// (feature_rule.hpp). Each candidate's xyz part is computed first, and its tails are loaded only when that part does
// not already exceed the best distance: the full distance can only be larger.
// Non-finite tails are inert: their distance is NaN or +inf and never passes d2 < bound.
#include "feature_rule.hpp"
#include "feature_search.cuh"
#include "grid_sweep.cuh"
#include "launch.cuh"

namespace cb {

namespace {

constexpr int kThreads = 256;

template <int NT>
__device__ __forceinline__ void load_tails(const float4* __restrict__ tails, uint32_t i, int kind, const Rigid* T,
                                           float* out) {
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    const float4 v = __ldg(tails + (size_t)i * NT + t);
    if (T && rule::tail_is_normal(kind, t)) {
      rule::rotate_tail(*T, v.x, v.y, v.z, out[3 * t], out[3 * t + 1], out[3 * t + 2]);
    } else {
      out[3 * t] = v.x;
      out[3 * t + 1] = v.y;
      out[3 * t + 2] = v.z;
    }
  }
}

template <int NT>
__global__ void feature_gather_kernel(int kind, const float4* __restrict__ pts, uint32_t n,
                                      const float4* __restrict__ raw, const Rigid T, bool rotate,
                                      float4* __restrict__ out) {
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    float v[3 * NT];
    load_tails<NT>(raw, (uint32_t)__float_as_int(__ldg(&pts[j].w)), kind, rotate ? &T : nullptr, v);
#pragma unroll
    for (int t = 0; t < NT; ++t) out[(size_t)j * NT + t] = make_float4(v[3 * t], v[3 * t + 1], v[3 * t + 2], 0.f);
  }
}

template <int NT>
__global__ void __launch_bounds__(kThreads) feature_nn_kernel(int kind, const GridView g,
                                                              const float4* __restrict__ g_tails,
                                                              const float4* __restrict__ q_pts, uint32_t n_q,
                                                              const float4* __restrict__ q_tails, const Rigid T,
                                                              bool rotate, float max_d2, int* __restrict__ out_idx,
                                                              float* __restrict__ out_d2) {
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n_q; k += gridDim.x * blockDim.x) {
    const float4 s = __ldg(q_pts + k);
    const uint32_t o = (uint32_t)__float_as_int(s.w);
    float qx, qy, qz;
    rule::transform_point(T, s.x, s.y, s.z, qx, qy, qz);
    float qt[3 * NT];
    load_tails<NT>(q_tails, o, kind, rotate ? &T : nullptr, qt);
    float best = max_d2;
    int best_idx = -1;
    grid_sweep(
        g, qx, qy, qz, [&]() { return best; },
        [&](uint32_t b, uint32_t e) {
          for (uint32_t j = b; j < e; ++j) {
            const float4 p = __ldg(g.pts + j);
            const float xyz = rule::contract_d2(qx, qy, qz, p.x, p.y, p.z);
            if (!(xyz <= best)) continue;  // feature_d2 >= xyz: cannot pass, nor tie
            float pt[3 * NT];
            load_tails<NT>(g_tails, j, kind, nullptr, pt);
            const float d2 = rule::feature_d2<NT>(xyz, qt, pt);
            const int pi = __float_as_int(p.w);
            if (d2 < best || (d2 == best && pi < best_idx)) {
              best = d2;
              best_idx = pi;
            }
          }
        },
        // the far sweep restarts on the block list: the best found so far is kept (a 1-NN with the index rule is
        // unchanged by meeting a candidate twice) and prunes the blocks from the start
        [&]() {},
        0u);  // k_needed = 0: the far sweep's xyz radius bound does not bound the feature-nearest point
    out_idx[o] = best_idx;
    out_d2[o] = best;
  }
}

}  // namespace

int launch_feature_gather(cb_context* ctx, int kind, const float4* pts, uint32_t n, const float4* raw, const Rigid* T,
                          float4* out) {
  if (n == 0) return CB_OK;
  const Rigid Tv = T ? *T : rigid_from_t12(nullptr);
  auto kernel = rule::feature_tails(kind) == 2 ? feature_gather_kernel<2> : feature_gather_kernel<1>;
  return launch(ctx, kernel, grid_for(ctx, n, kThreads, 16), kThreads, 0, kind, pts, n, raw, Tv, T != nullptr, out);
}

int launch_feature_nn(cb_context* ctx, int kind, const GridView& g, const float4* g_tails, const float4* q_pts,
                      uint32_t n_q, const float4* q_tails, const Rigid& T, bool rotate, float max_d2, int* out_idx,
                      float* out_d2) {
  if (n_q == 0) return CB_OK;
  auto kernel = rule::feature_tails(kind) == 2 ? feature_nn_kernel<2> : feature_nn_kernel<1>;
  return launch(ctx, kernel, grid_for(ctx, n_q, kThreads, 16), kThreads, 0, kind, g, g_tails, q_pts, n_q, q_tails, T,
                rotate, max_d2, out_idx, out_d2);
}

}  // namespace cb
