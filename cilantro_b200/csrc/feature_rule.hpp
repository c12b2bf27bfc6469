// Feature-space correspondence distance of the rigid ICP (product code, host and device).
//
// Replaces the feature adaptors of correspondence_search/common_transformable_feature_adaptors.hpp (PointNormal /
// PointColor / PointNormalColor, :148-290) and the L2 metric nanoflann evaluates on them (L2_Adaptor::evalMetric,
// nanoflann.hpp:570-604). A feature is xyz followed by one or two 3-vector TAILS: w_n n (normal part) and / or w_c c
// (colour part), formed once at upload with one fp32 multiply per component (the adaptors' constructors, :175-183,
// :248-259). feature_search.cu compiles this header for the device; tests/cpp/test_feature_rule.cpp for the host
// (-ffp-contract=off), against the reference's own evalMetric.
//
// Arithmetic (fp32, one rounding per operation, no FMA): d_k = q_k - p_k, and evalMetric's order — groups of four
// components ((d0² + d1²) + d2²) + d3² added to the running sum while four remain, the rest one at a time:
//   D = 3  ((d0² + d1²) + d2²)                              = contract_d2 (cache_rule.hpp)
//   D = 6  ((g(0..3) + d4²) + d5²)
//   D = 9  ((g(0..3) + g(4..7)) + d8²)
// (the running sum starts at +0, and 0 + g = g exactly). evalMetric may return early once the partial sum exceeds the
// current worst distance; that partial sum already fails the strict acceptance test d2 < worst, and so would the full
// sum (it is never smaller), so the early return cannot change an accept / reject decision.
//
// Exactness of the 3-D grid for this distance: g(0..3) = contract_d2(xyz) + d3², and a round-to-nearest addition of a
// non-negative term never decreases a sum, so feature_d2 >= contract_d2(xyz part) for every input (NaN compares false
// either way). Every lower bound the grid searches derive from the xyz distance (shell walk, slab / open-face gaps,
// far-sweep block bounds) is therefore a lower bound of the feature distance too. The radius bound of the far sweep is
// NOT: the xyz-nearest block says nothing about the feature-nearest point, so feature searches run it with k_needed = 0.
#pragma once
#include "cache_rule.hpp"

namespace cb {
namespace rule {

// = cb_feature_kind of the C ABI
enum FeatureKind : int { kFeatPoint = 0, kFeatPointNormal = 1, kFeatPointColor = 2, kFeatPointNormalColor = 3 };

// number of 3-vector tails after xyz
CB_RULE_HD int feature_tails(int kind) { return kind == kFeatPointNormalColor ? 2 : (kind == kFeatPoint ? 0 : 1); }

// tail i of a feature of this kind is a normal (rotated by the transform) rather than a colour (copied)
CB_RULE_HD bool tail_is_normal(int kind, int i) { return i == 0 && (kind == kFeatPointNormal || kind == kFeatPointNormalColor); }

// R (w n) with transform_point's per-row arithmetic, without the translation: transformFeatures, Isometry branch
// (:193-204, :269-280)
template <class RigidT>
CB_RULE_HD void rotate_tail(const RigidT& T, float x, float y, float z, float& ox, float& oy, float& oz) {
  ox = add_rn(mul_rn(T.r[0], x), add_rn(mul_rn(T.r[1], y), mul_rn(T.r[2], z)));
  oy = add_rn(mul_rn(T.r[3], x), add_rn(mul_rn(T.r[4], y), mul_rn(T.r[5], z)));
  oz = add_rn(mul_rn(T.r[6], x), add_rn(mul_rn(T.r[7], y), mul_rn(T.r[8], z)));
}

CB_RULE_HD float sq_diff(float a, float b) {
  const float d = sub_rn(a, b);
  return mul_rn(d, d);
}

// The feature distance from its xyz part xyz_d2 = contract_d2(q_xyz, p_xyz) and the TAILS * 3 tail components of the
// query (q) and the reference point (p).
template <int TAILS>
CB_RULE_HD float feature_d2(float xyz_d2, const float* q, const float* p) {
  if (TAILS == 0) return xyz_d2;
  float d = add_rn(xyz_d2, sq_diff(q[0], p[0]));  // g(0..3)
  if (TAILS == 1) {
    d = add_rn(d, sq_diff(q[1], p[1]));
    return add_rn(d, sq_diff(q[2], p[2]));
  }
  float g = add_rn(sq_diff(q[1], p[1]), sq_diff(q[2], p[2]));  // g(4..7)
  g = add_rn(g, sq_diff(q[3], p[3]));
  g = add_rn(g, sq_diff(q[4], p[4]));
  d = add_rn(d, g);
  return add_rn(d, sq_diff(q[5], p[5]));
}

}  // namespace rule
}  // namespace cb
