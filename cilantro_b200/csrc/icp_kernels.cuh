// Kernel-side declarations for the fused ICP iteration (product code).
#pragma once
#include "cb_internal.hpp"
#include "nn_search.cuh"
#include "projection.hpp"

namespace cb {

enum IcpMode : int {
  kModeKnn = 0,       // per-query nearest neighbour only (cb_knn1_radius / correspondences)
  kModeP2P = 1,       // Kabsch moments: n, sum d, sum q, sum d q^T                       (16 values)
  kModeCombined = 2,  // Gauss-Newton normal equations: n, upper AtA (21), Atb (6)         (28 values)
  kModeP2PCentered = 3,  // Kabsch moments about the pivots (dst mean, T * src mean): what both ICP loops accumulate
};

constexpr int kP2PValues = 16;
constexpr int kCombinedValues = 28;
constexpr int kMaxValues = 28;

struct IcpArgs {
  GridView dst;
  const float4* src_pts;  // cell-sorted query cloud; .w = original index bits
  const float4* src_nrm;  // same order, or nullptr (symmetric metric when set)
  uint32_t n_src;
  Rigid T;       // current estimate: q = T * s  (the search AND the estimator use this q)
  Rigid Tin;     // inner Gauss-Newton transform (identity in the fused first pass)
  float max_d2;
  uint32_t prefetch_blocks;  // L2 prefetch look-ahead of the search kernel, in blocks (set by the launcher)
  float w_pt, w_pl;
  int wk_pt, wk_pl;     // cb_weight_kind of the two correspondence weight evaluators
  float wc_pt, wc_pl;   // RBF coefficients -0.5 / sigma^2
  float dm[3];   // dst_mean_
  float sm[3];   // transform_ * src_mean_
  // per-query results, indexed by position in the SORTED query cloud (nullable)
  const int* warm_pos;  // previous iteration's nn_pos (same layout) or nullptr: seeds the search (warp_search.cuh)
  int* nn_pos;    // position of the match in the sorted dst cloud, -1 = none
  float* nn_d2;   // its squared distance
  // per-query results in ORIGINAL query order (kModeKnn; nullable)
  int* out_idx;   // original dst index or -1
  float* out_d2;
  // reduction scratch
  ReduceScratch rs;  // grid-reduction scratch (set by the launcher)
};

// One pass over the query cloud. kSearch = false re-uses nn_pos from a previous pass (inner
// Gauss-Newton iterations >= 2 keep the correspondences fixed, transform_estimation.hpp:281).
int launch_icp_pass(cb_context* ctx, const IcpArgs& a, int mode, bool search, bool has_pt, bool has_pl);

// Accumulation over an explicit correspondence list (non-default engine modes, icp_engine.cu): pair p =
// (dst point first[p], src point second[p]) by ORIGINAL index; a supplies T, Tin, dm, sm, w_pt, w_pl.
int launch_pairs_pass(cb_context* ctx, const IcpArgs& a, const EnginePairs& pairs, const cb_cloud* dst,
                      const cb_cloud* src, int mode, bool has_pt, bool has_pl);

// computeResiduals: unbounded 1-NN + the weighted residual, original query order.
int launch_residuals(cb_context* ctx, const GridView& dst, const float4* src_pts, const float4* src_nrm,
                     uint32_t n_src, const Rigid& T, int metric, float w_pt, float w_pl, float* d_out);

int launch_transform_points(cb_context* ctx, const Rigid& T, const float* d_in, size_t n, float* d_out);

// Per sorted source position p: out_first[orig(p)] = original index of dst point nn_pos[p] (or -1),
// out_val[orig(p)] = nn_d2[p] (nullable) - the getters' translation from sorted positions to caller indices.
int launch_translate_matches(cb_context* ctx, const int* nn_pos, const float* nn_d2, const float4* src_pts,
                             const float4* dst_pts, uint32_t n_src, int* out_first, float* out_val);

// Projective correspondence search (projective_search.cu). Per source point of the cloud src_pts (.w = original index
// bits), under T: nn_pos / nn_d2 by position in src_pts (the destination's sorted position, -1 none), out_idx / out_d2
// by original index (the destination's original index, -1 none); every output is nullable.
int launch_projective_search(cb_context* ctx, const ProjectiveMap& pm, const float4* src_pts, uint32_t n_src,
                             const float4* dst_pts, const Rigid& T, float max_d2, int* nn_pos, float* nn_d2,
                             int* out_idx, float* out_d2);
// The index map of the projection (K9 row-major 3 x 3, E12 row-major [R | t] or nullptr, w x h pixels) over the indexed
// cloud dst, into *out (on, its d_map owned by `owner`). Non-finite K or E, or w * h >= 2^32, give CB_ERR_INVALID; on
// any error *out is untouched and nothing stays allocated. Synchronises the stream.
int build_projective_map(cb_context* ctx, DeviceScope& owner, const cb_cloud* dst, const float* K9, size_t w, size_t h,
                         const float* E12, ProjectiveMap* out);

}  // namespace cb
