// ORACLE — test infrastructure, NOT product code.
// Serial restatement of RandomSampleConsensusBase::estimate (model_estimation/ransac_base.hpp:64-131) with
// HyperplaneRANSACEstimator<float, 3> (model_estimation/ransac_hyperplane_estimator.hpp), DESIGN §4.12: built by
// oracle/Makefile into oracle/libplane_oracle.so with -ffp-contract=off.
//
// Hypothesis plane of a sample: the closed form pinned in DESIGN §4.12 (double, one rounding per operation). Residual:
// |((n0 x) + ((n1 y) + (n2 z))) + d| in fp32. Re-estimation: the PCA of the kept hypothesis's inliers with the
// reference's fp32 serial sums (covariance.hpp:64-76), or double sums with accum_double; eigenvectors from the
// double Jacobi of small_linalg.hpp (Eigen's solver is unpinned, DESIGN §6).
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <limits>
#include <random>
#include <utility>
#include <vector>

#include "small_linalg.hpp"

#define ORC_API extern "C" __attribute__((visibility("default")))

namespace {

const float kNaN = std::numeric_limits<float>::quiet_NaN();

void cross(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}
double sqnorm(const double* v) { return v[0] * v[0] + (v[1] * v[1] + v[2] * v[2]); }
void unit(const double* v, double* n) {
  const double s = std::sqrt(sqnorm(v));
  for (int r = 0; r < 3; r++) n[r] = v[r] / s;
}
// a plane containing the line along u: normalize(u x e_k), k = argmin |u_k| (lowest k on ties); u = 0: (0, 0, 1)
void line_normal(const double* u, double* n) {
  if (sqnorm(u) == 0.0) {
    n[0] = 0.0, n[1] = 0.0, n[2] = 1.0;
    return;
  }
  int k = 0;
  if (std::fabs(u[1]) < std::fabs(u[k])) k = 1;
  if (std::fabs(u[2]) < std::fabs(u[k])) k = 2;
  double e[3] = {0.0, 0.0, 0.0}, c[3];
  e[k] = 1.0;
  cross(u, e, c);
  unit(c, n);
}

}  // namespace

// estimateModel(sample) for a sample of `count` points (packed xyz): plane (n0, n1, n2, d)
ORC_API void orc_plane_fit(const float* p, int count, float* out) {
  bool finite = count >= 2;
  for (int i = 0; i < 3 * count && i < 9; i++) finite = finite && std::isfinite(p[i]);
  if (!finite) {  // covariance.hpp:35 (fewer than 2 points), or a non-finite sample point
    for (int r = 0; r < 4; r++) out[r] = kNaN;
    return;
  }
  double q[3][3] = {};
  for (int i = 0; i < count && i < 3; i++)
    for (int r = 0; r < 3; r++) q[i][r] = p[3 * i + r];
  double n[3], m[3];
  if (count == 2) {
    const double u[3] = {q[1][0] - q[0][0], q[1][1] - q[0][1], q[1][2] - q[0][2]};
    line_normal(u, n);
    for (int r = 0; r < 3; r++) m[r] = (q[0][r] + q[1][r]) / 2.0;
  } else {
    double a[3], b[3], e[3], c[3];
    for (int r = 0; r < 3; r++) {
      a[r] = q[1][r] - q[0][r];
      b[r] = q[2][r] - q[0][r];
      e[r] = q[2][r] - q[1][r];
    }
    cross(a, b, c);
    if (c[0] != 0.0 || c[1] != 0.0 || c[2] != 0.0) {
      unit(c, n);
    } else {  // collinear or coincident: the longest of a, b, p2 - p1, the first on ties
      const double* u = a;
      if (sqnorm(b) > sqnorm(u)) u = b;
      if (sqnorm(e) > sqnorm(u)) u = e;
      line_normal(u, n);
    }
    for (int r = 0; r < 3; r++) m[r] = ((q[0][r] + q[1][r]) + q[2][r]) / 3.0;
  }
  const double d = -(n[0] * m[0] + (n[1] * m[1] + n[2] * m[2]));
  for (int r = 0; r < 3; r++) out[r] = (float)n[r];
  out[3] = (float)d;
}

static inline float residual(const float* pl, const float* p) {
  return std::fabs((pl[0] * p[0] + (pl[1] * p[1] + pl[2] * p[2])) + pl[3]);
}

// computeResiduals (:47-55) + the serial scan (ransac_base.hpp:96-101); residuals / inliers may be null
ORC_API size_t orc_plane_residuals(const float* pts, size_t n, const float* plane, float thresh, float* residuals,
                                   uint64_t* inliers) {
  size_t k = 0;
  for (size_t i = 0; i < n; i++) {
    const float r = residual(plane, pts + 3 * i);
    if (residuals) residuals[i] = r;
    if (r <= thresh) {
      if (inliers) inliers[k] = i;
      k++;
    }
  }
  return k;
}

ORC_API void orc_plane_score(const float* pts, size_t n, const float* planes, size_t H, float thresh,
                             uint32_t* counts) {
#pragma omp parallel for schedule(dynamic, 1)
  for (size_t h = 0; h < H; h++) counts[h] = (uint32_t)orc_plane_residuals(pts, n, planes + 4 * h, thresh, nullptr, nullptr);
}

// PrincipalComponentAnalysis<float, 3>(points, subset) (core/principal_component_analysis.hpp:24-30, :76-84) and
// the plane of estimate_params_ (ransac_hyperplane_estimator.hpp:103-110): normal = the third eigenvector column
// after the determinant fix, offset = -(normal . mean) in fp32
ORC_API void orc_plane_pca(const float* pts, const uint64_t* idx, size_t m, int accum_double, float* out) {
  if (m < 2) {
    for (int r = 0; r < 4; r++) out[r] = kNaN;
    return;
  }
  float mean[3], cov[9];
  if (!accum_double) {  // covariance.hpp:64-76, fp32 serial
    float ms[3] = {0, 0, 0};
    for (size_t i = 0; i < m; i++)
      for (int r = 0; r < 3; r++) ms[r] += pts[3 * idx[i] + r];
    const float inv = 1.0f / (float)m;
    for (int r = 0; r < 3; r++) mean[r] = inv * ms[r];
    float cs[9] = {0};
    for (size_t i = 0; i < m; i++) {
      const float* p = pts + 3 * idx[i];
      const float t[3] = {p[0] - mean[0], p[1] - mean[1], p[2] - mean[2]};
      for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) cs[r * 3 + c] += t[r] * t[c];
    }
    const float inv1 = 1.0f / (float)(m - 1);
    for (int i = 0; i < 9; i++) cov[i] = inv1 * cs[i];
  } else {
    double ms[3] = {0, 0, 0};
    for (size_t i = 0; i < m; i++)
      for (int r = 0; r < 3; r++) ms[r] += pts[3 * idx[i] + r];
    double mu[3];
    for (int r = 0; r < 3; r++) {
      mu[r] = ms[r] / (double)m;
      mean[r] = (float)mu[r];
    }
    double cs[9] = {0};
    for (size_t i = 0; i < m; i++) {
      const float* p = pts + 3 * idx[i];
      const double t[3] = {p[0] - mu[0], p[1] - mu[1], p[2] - mu[2]};
      for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) cs[r * 3 + c] += t[r] * t[c];
    }
    for (int i = 0; i < 9; i++) cov[i] = (float)(cs[i] / (double)(m - 1));
  }
  orc::M3 C, V;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) C.a[r][c] = cov[r * 3 + c];
  double w[3];
  orc::sym3_eigen(C, w, V);  // ascending
  orc::M3 E;                 // descending columns
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) E.a[r][c] = V.a[r][2 - c];
  if (orc::m3_det(E) < 0.0)
    for (int r = 0; r < 3; r++) E.a[r][2] = -E.a[r][2];
  const float n[3] = {(float)E.a[0][2], (float)E.a[1][2], (float)E.a[2][2]};
  for (int r = 0; r < 3; r++) out[r] = n[r];
  out[3] = -(n[0] * mean[0] + (n[1] * mean[1] + n[2] * mean[2]));
}

// the first `iters` samples (sample_size = min(3, n)) and their planes, as the loop draws them
ORC_API void orc_plane_hypotheses(const float* pts, size_t n, uint32_t seed, size_t iters, uint64_t* samples,
                                  float* planes) {
  const size_t ss = n < 3 ? n : 3;
  std::vector<size_t> perm(n);
  for (size_t i = 0; i < n; i++) perm[i] = i;
  std::mt19937 rng(seed);
  for (size_t it = 0; it < iters; it++) {
    size_t prev = n;
    float p[9];
    for (size_t i = 0; i < ss; i++) {
      std::uniform_int_distribution<size_t> dist(0, prev - 1);
      const size_t r = dist(rng);
      samples[3 * it + i] = perm[r];
      for (int c = 0; c < 3; c++) p[3 * i + c] = pts[3 * perm[r] + c];
      prev--;
      std::swap(perm[r], perm[prev]);
    }
    orc_plane_fit(p, (int)ss, planes + 4 * it);
  }
}

struct orc_plane_result {
  float plane[4];
  float hyp_plane[4];
  uint64_t iterations;
  uint64_t best_iteration;
  uint64_t num_inliers;
};

ORC_API void orc_ransac_plane(const float* pts, size_t n, uint32_t seed, size_t inlier_count_thresh, size_t max_iter,
                              float thresh, int re_estimate, int accum_double, orc_plane_result* out,
                              uint64_t* inliers /* n */, float* residuals /* n */) {
  size_t sample_size = 3;
  if (n < sample_size) sample_size = n;                  // :67
  if (inlier_count_thresh > n) inlier_count_thresh = n;  // :68
  std::vector<size_t> perm(n);
  for (size_t i = 0; i < n; i++) perm[i] = i;
  std::mt19937 rng(seed);
  float best[4] = {kNaN, kNaN, kNaN, kNaN};  // stand-in for the uninitialised Eigen::Hyperplane
  std::vector<uint64_t> best_inl, cur_inl(n);
  size_t it = 0, best_it = 0;
  while (it < max_iter) {
    float p[9];
    size_t prev = n;
    for (size_t i = 0; i < sample_size; i++) {  // :83-91
      std::uniform_int_distribution<size_t> dist(0, prev - 1);
      const size_t r = dist(rng);
      for (int c = 0; c < 3; c++) p[3 * i + c] = pts[3 * perm[r] + c];
      prev--;
      std::swap(perm[r], perm[prev]);
    }
    float cur[4];
    orc_plane_fit(p, (int)sample_size, cur);  // :94
    cur_inl.resize(n);
    const size_t k = orc_plane_residuals(pts, n, cur, thresh, nullptr, cur_inl.data());  // :95-101
    cur_inl.resize(k);
    it++;
    if (k < sample_size) continue;  // :104
    if (k > best_inl.size()) {      // :107-111
      std::memcpy(best, cur, sizeof(best));
      best_inl = cur_inl;
      best_it = it - 1;
    }
    if (best_inl.size() >= inlier_count_thresh) break;  // :114
  }
  float plane[4];
  std::memcpy(plane, best, sizeof(plane));
  if (re_estimate && !best_inl.empty()) orc_plane_pca(pts, best_inl.data(), best_inl.size(), accum_double, plane);
  std::memcpy(out->plane, plane, sizeof(plane));
  std::memcpy(out->hyp_plane, best, sizeof(best));
  out->iterations = it;
  out->best_iteration = best_it;
  out->num_inliers = orc_plane_residuals(pts, n, plane, thresh, residuals, inliers);
}
