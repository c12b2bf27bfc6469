// ORACLE — test infrastructure, NOT product code.
// Serial restatement of extractConnectedComponents in its neighbourhood-set form (clustering/
// connected_component_extraction.hpp:21-118; the kd-tree form :163-265 runs the same logic on tree.search() results)
// and of the proximity evaluators (core/common_pair_evaluators.hpp:88-259). Built by oracle/Makefile into
// oracle/libcce_oracle.so; compile with -ffp-contract=off (the arithmetic contract of cilantro_oracle.cpp).
//
// Restated for ONE thread: the reference's OpenMP seed loop (:36-65) shares current_label without synchronisation.
// The final std::sort (:117) is a std::stable_sort here, which pins the order of equal-size segments (DESIGN §6).
// Neighbourhoods come from the caller, ascending (d2, index) (BruteKnn, or the reference nanoflann re-sorted on that
// key). The angle test evaluates std::acos itself: it shares nothing with the product's threshold derivation.
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <limits>
#include <set>
#include <vector>

#define ORC_API extern "C" __attribute__((visibility("default")))

namespace {

struct Eval {
  int terms;  // 1 points, 2 normals, 4 colours; 0 = AlwaysTrueEvaluator
  int strict;
  float max_distance, max_angle, max_color_diff;
  const float* normals;
  const float* colors;

  // Eigen 3-term dot: a0 + (a1 + a2)
  static float dot(const float* a, const float* b) { return a[0] * b[0] + (a[1] * b[1] + a[2] * b[2]); }

  bool angle_ok(size_t i, size_t j) const {
    const float angle = std::acos(dot(normals + 3 * i, normals + 3 * j));
    if (max_angle >= 0.0f) return strict ? angle < max_angle : angle <= max_angle;
    return strict ? std::min(angle, (float)M_PI - angle) < -max_angle
                  : std::min(angle, (float)M_PI - angle) <= -max_angle;
  }
  bool color_ok(size_t i, size_t j) const {
    const float d[3] = {colors[3 * i] - colors[3 * j], colors[3 * i + 1] - colors[3 * j + 1],
                        colors[3 * i + 2] - colors[3 * j + 2]};
    return dot(d, d) < max_color_diff;
  }
  // the reference's classes, terms in their order
  bool operator()(size_t i, size_t j, float dist) const {
    switch (terms) {
      case 0: return true;                                  // AlwaysTrueEvaluator (:86)
      case 1: return dist < max_distance;                   // PointsProximityEvaluator (:97)
      case 2: return angle_ok(i, j);                        // NormalsProximityEvaluator (:114-121)
      case 4: return color_ok(i, j);                        // ColorsProximityEvaluator (:138-140)
      case 3:                                               // PointsNormalsProximityEvaluator (:158-166)
        if (dist >= max_distance) return false;
        return angle_ok(i, j);
      case 5:                                               // PointsColorsProximityEvaluator (:184-187)
        return (dist < max_distance) && color_ok(i, j);
      case 6:                                               // NormalsColorsProximityEvaluator (:210-218)
        if (!color_ok(i, j)) return false;
        return angle_ok(i, j);
      default:                                              // PointsNormalsColorsProximityEvaluator (:243-252)
        if (dist >= max_distance || !color_ok(i, j)) return false;
        return angle_ok(i, j);
    }
  }
};

}  // namespace

// idx / d2: n rows of `stride` entries, cnt[p] valid per row (= N(p), ascending (d2, index)). seeds == NULL: every
// point, in index order. Outputs: p2c[n], offsets[m + 1], points[offsets[m]]; returns m.
ORC_API size_t orc_connected_components(size_t n, const int64_t* idx, const float* d2, size_t stride,
                                        const uint32_t* cnt, const uint64_t* seeds, size_t n_seeds, int terms,
                                        int strict, float max_distance, float max_angle, float color_thresh,
                                        const float* normals, const float* colors, uint64_t min_segment_size,
                                        uint64_t max_segment_size, uint64_t* p2c, uint64_t* offsets,
                                        uint64_t* points) {
  Eval evaluator{terms, strict, max_distance, max_angle, color_thresh * color_thresh, normals, colors};
  std::vector<uint64_t> seeds_ind;
  if (seeds) {
    seeds_ind.assign(seeds, seeds + n_seeds);
  } else {
    seeds_ind.resize(n);
    for (size_t i = 0; i < n; i++) seeds_ind[i] = i;
  }
  // :26-34
  constexpr size_t unassigned = std::numeric_limits<size_t>::max();
  std::vector<size_t> current_label(n, unassigned);
  std::vector<size_t> frontier_set;
  frontier_set.reserve(n);
  std::vector<std::set<size_t>> seeds_to_merge_with(seeds_ind.size());
  std::vector<char> seed_active(seeds_ind.size(), 0);
  // :36-65, one thread
  for (size_t i = 0; i < seeds_ind.size(); i++) {
    if (current_label[seeds_ind[i]] != unassigned) continue;
    seeds_to_merge_with[i].insert(i);
    frontier_set.clear();
    frontier_set.emplace_back(seeds_ind[i]);
    current_label[seeds_ind[i]] = i;
    seed_active[i] = 1;
    while (!frontier_set.empty()) {
      const size_t curr_seed = frontier_set.back();
      frontier_set.pop_back();
      const int64_t* nn_idx = idx + curr_seed * stride;
      const float* nn_val = d2 + curr_seed * stride;
      for (size_t j = 1; j < cnt[curr_seed]; j++) {
        const size_t curr_lbl = current_label[nn_idx[j]];
        if (curr_lbl != i && evaluator(curr_seed, nn_idx[j], nn_val[j])) {
          if (curr_lbl == unassigned) {
            frontier_set.emplace_back(nn_idx[j]);
            current_label[nn_idx[j]] = i;
          } else {
            seeds_to_merge_with[i].insert(curr_lbl);
          }
        }
      }
    }
  }
  // :67-71
  for (size_t i = 0; i < seeds_to_merge_with.size(); i++) {
    for (auto it = seeds_to_merge_with[i].begin(); it != seeds_to_merge_with[i].end(); ++it) {
      seeds_to_merge_with[*it].insert(i);
    }
  }
  // :73-95
  std::vector<size_t> seed_repr(seeds_ind.size(), unassigned);
  size_t seed_cluster_num = 0;
  for (size_t i = 0; i < seeds_to_merge_with.size(); i++) {
    if (seed_active[i] == 0 || seed_repr[i] != unassigned) continue;
    frontier_set.clear();
    frontier_set.emplace_back(i);
    seed_repr[i] = seed_cluster_num;
    while (!frontier_set.empty()) {
      const size_t curr_seed = frontier_set.back();
      frontier_set.pop_back();
      for (auto it = seeds_to_merge_with[curr_seed].begin(); it != seeds_to_merge_with[curr_seed].end(); ++it) {
        if (seed_active[i] == 1 && seed_repr[*it] == unassigned) {
          frontier_set.emplace_back(*it);
          seed_repr[*it] = seed_cluster_num;
        }
      }
    }
    seed_cluster_num++;
  }
  // :97-104 (a segment stops growing at max + 1 points)
  std::vector<std::vector<uint64_t>> segment_to_point_map_tmp(seed_cluster_num);
  for (size_t i = 0; i < current_label.size(); i++) {
    if (current_label[i] == unassigned) continue;
    const auto ind = seed_repr[current_label[i]];
    if (segment_to_point_map_tmp[ind].size() <= max_segment_size) segment_to_point_map_tmp[ind].emplace_back(i);
  }
  // :106-113
  std::vector<std::vector<uint64_t>> segment_to_point_map;
  for (size_t i = 0; i < segment_to_point_map_tmp.size(); i++) {
    if (segment_to_point_map_tmp[i].size() >= min_segment_size &&
        segment_to_point_map_tmp[i].size() <= max_segment_size) {
      segment_to_point_map.emplace_back(std::move(segment_to_point_map_tmp[i]));
    }
  }
  // :115-117, stable
  std::stable_sort(segment_to_point_map.begin(), segment_to_point_map.end(),
                   [](const std::vector<uint64_t>& a, const std::vector<uint64_t>& b) { return a.size() > b.size(); });
  // getPointToClusterIndexMap (clustering_base.hpp:8-17) and the CSR of the cluster -> points map
  const size_t m = segment_to_point_map.size();
  for (size_t i = 0; i < n; i++) p2c[i] = m;
  size_t o = 0;
  for (size_t c = 0; c < m; c++) {
    offsets[c] = o;
    for (uint64_t p : segment_to_point_map[c]) {
      p2c[p] = c;
      points[o++] = p;
    }
  }
  offsets[m] = o;
  return m;
}
