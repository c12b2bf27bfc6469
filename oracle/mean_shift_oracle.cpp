// ORACLE — test infrastructure, NOT product code.
// Serial restatement of MeanShift<float, 3>::cluster (clustering/mean_shift.hpp:37-115) for the fp32 arithmetic
// contract of cilantro_oracle.cpp: built by oracle/Makefile into oracle/libms_oracle.so with -ffp-contract=off.
//
// Neighbourhoods: a brute-force radius search with BruteKnn's arithmetic (d2 = ((dx^2 + dy^2) + dz^2), dx = q - p,
// strict d2 < r2), sorted on (d2, index), which pins the order the reference leaves to std::sort (DESIGN §6). The
// seeds are independent (the reference's OpenMP seed loop, :57), so they are shifted in parallel here too; every
// seed's arithmetic is serial and in list order.
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <utility>
#include <vector>

#define ORC_API extern "C" __attribute__((visibility("default")))

namespace {

// radiusSearch(q, r2, nn) (core/kd_tree.hpp:250-278), ascending (d2, index)
void radius_search(const float* pts, size_t n, const float* q, float r2, std::vector<std::pair<float, size_t>>& nn) {
  nn.clear();
  for (size_t j = 0; j < n; j++) {
    const float dx = q[0] - pts[3 * j], dy = q[1] - pts[3 * j + 1], dz = q[2] - pts[3 * j + 2];
    const float d2 = (dx * dx + dy * dy) + dz * dz;
    if (d2 < r2) nn.emplace_back(d2, j);
  }
  std::sort(nn.begin(), nn.end());
}

float sq_dist(const float* a, const float* b) {  // (a - b).squaredNorm()
  const float dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
  return (dx * dx + dy * dy) + dz * dz;
}

}  // namespace

// pts: n x 3; seeds: ns x 3 (the cloud's points for the all-points overload, :118-124). rbf != 0:
// RBFKernelWeightEvaluator<float, float, true> with coefficient coeff (core/common_pair_evaluators.hpp:46-79), else
// UnityWeightEvaluator. Outputs sized by ns: shifted[3 ns], p2c[ns], offsets[ns + 1], members[ns], modes[3 ns];
// *num_clusters. Returns getNumberOfPerformedIterations().
ORC_API uint64_t orc_mean_shift(size_t n, const float* pts, size_t ns, const float* seeds, float kernel_radius,
                                uint64_t max_iter, float cluster_tol, float convergence_tol, int rbf, float coeff,
                                float* shifted, uint64_t* p2c, uint64_t* offsets, uint64_t* members, float* modes,
                                size_t* num_clusters) {
  std::copy(seeds, seeds + 3 * ns, shifted);  // :43
  // :46-48
  const float radius_sq = kernel_radius * kernel_radius;
  const float conv_tol_sq = convergence_tol * convergence_tol;
  uint64_t iteration_count = 0;
  std::vector<char> has_converged(ns, 0);
  // :55-82
  while (iteration_count < max_iter) {
    bool all_converged = true;
#pragma omp parallel for schedule(dynamic, 1) reduction(&& : all_converged)
    for (size_t i = 0; i < ns; i++) {
      if (has_converged[i]) continue;
      std::vector<std::pair<float, size_t>> nn;
      float* s = shifted + 3 * i;
      radius_search(pts, n, s, radius_sq, nn);
      float point_tmp[3] = {0.0f, 0.0f, 0.0f};
      float total_weight = 0.0f;
      for (size_t j = 0; j < nn.size(); j++) {
        const float weight = rbf ? std::exp(coeff * nn[j].first) : 1.0f;  // evaluator(seed, point, d2)
        const float* p = pts + 3 * nn[j].second;
        for (int c = 0; c < 3; c++) point_tmp[c] += weight * p[c];
        total_weight += weight;
      }
      const float inv = 1.0f / total_weight;  // :70
      for (int c = 0; c < 3; c++) point_tmp[c] *= inv;
      if (sq_dist(s, point_tmp) < conv_tol_sq) {
        has_converged[i] = 1;
      } else {
        all_converged = false;
      }
      for (int c = 0; c < 3; c++) s[c] = point_tmp[c];
    }
    iteration_count++;
    if (all_converged) break;
  }
  // :84-100
  const float cluster_tol_sq = cluster_tol * cluster_tol;
  std::vector<std::vector<uint64_t>> clusters;
  for (size_t i = 0; i < ns; i++) {
    size_t c;
    for (c = 0; c < clusters.size(); c++) {
      if (sq_dist(shifted + 3 * i, shifted + 3 * clusters[c][0]) < cluster_tol_sq) break;
    }
    if (c == clusters.size()) {
      clusters.emplace_back(1, i);
    } else {
      clusters[c].emplace_back(i);
    }
  }
  // :102-112, and the CSR of the cluster -> seeds map
  size_t o = 0;
  for (size_t c = 0; c < clusters.size(); c++) {
    float m[3] = {0.0f, 0.0f, 0.0f};
    offsets[c] = o;
    for (uint64_t i : clusters[c]) {
      for (int k = 0; k < 3; k++) m[k] += shifted[3 * i + k];
      p2c[i] = c;
      members[o++] = i;
    }
    const float inv = 1.0f / (float)clusters[c].size();
    for (int k = 0; k < 3; k++) modes[3 * c + k] = m[k] * inv;
  }
  offsets[clusters.size()] = o;
  *num_clusters = clusters.size();
  return iteration_count;
}
