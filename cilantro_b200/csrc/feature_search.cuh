// Feature-space 1-NN over the uniform grid (feature_search.cu): declarations for the ICP's list path.
#pragma once
#include "cb_internal.hpp"
#include "nn_search.cuh"

namespace cb {

// out[j * tails + t] = tail t of the point at cell-sorted position j of `pts` (its original index in .w), taken from
// `raw` (original order, `tails` float4 per point). T != nullptr rotates the normal tail (transformFeatures), as the
// grid over {T src} of FIRST_TO_SECOND needs; nullptr copies.
int launch_feature_gather(cb_context* ctx, int kind, const float4* pts, uint32_t n, const float4* raw, const Rigid* T,
                          float4* out);

// Radius-bounded feature 1-NN (rule::feature_d2, d2 < max_d2, exact ties -> lowest original index) of every query of
// the cell-sorted cloud q_pts, transformed by T, with tails q_tails (original query order; the normal tail rotated by T
// when `rotate`), among the points of grid g whose tails are g_tails (g's cell order). Results in original query order:
// out_idx = original reference index or -1, out_d2 = its feature d2.
int launch_feature_nn(cb_context* ctx, int kind, const GridView& g, const float4* g_tails, const float4* q_pts,
                      uint32_t n_q, const float4* q_tails, const Rigid& T, bool rotate, float max_d2, int* out_idx,
                      float* out_d2);

}  // namespace cb
