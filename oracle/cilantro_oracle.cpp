// ORACLE — test infrastructure, NOT product code.
//
// CPU restatement (no Eigen, no CUDA) of the rigid-ICP / k-means / RANSAC / PCA hot path of
// kzampog/cilantro, written from the reference's behaviour; every function cites the
// reference file:line it follows (paths relative to the reference's include/cilantro/).
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
// load this library, and only as the checker / CPU baseline. The product
// (cilantro_b200/csrc) never links, includes or calls anything in oracle/.
//
// PARITY PINNING. The reference ships no tests or golden vectors (SURVEY.md F2). What pins
// this restatement:
//   * kNN: the reference's own vendored nanoflann 1.7.1, compiled in place into
//     oracle/_ref/ (oracle/nanoflann_ref.cpp) — orc_knn1_brute must agree with it on every
//     query (equal index, or bit-equal d2 on exact ties), see tests/test_oracle_kat.py
//     (test_brute_restatement_agrees_with_reference_nanoflann); the full-size runs of BASELINE's configs 2 and 3
//     (tests/test_gpu_full_size.py) search with that reference nanoflann inside the restated loop;
//   * the correspondence-weight evaluators (Unity / RBFKernelWeightEvaluator, common_pair_evaluators.hpp:54-60) and
//     the weighted normal equations: an independent numpy restatement of transform_estimation.hpp:285-357
//     (tests/test_oracle_rbf.py);
//   * the hand-derivable known answers of examples/kd_tree.cpp and
//     examples/principal_component_analysis.cpp (tests/test_oracle_kat.py);
//   * the self-checking recipe of examples/rigid_icp.cpp (estimate ~= tf_ref^-1);
//   * the callers either side of the path (normal estimation, voxel-grid downsampling, the correspondence
//     engine's non-default modes): k-neighbourhoods and radius lists come from the reference nanoflann
//     (tests/test_oracle_normals.py, tests/golden/make_golden.py refuse a brute-force / nanoflann mismatch);
//     the per-neighbourhood covariance, the std::map grid accumulation and the sort / set_union /
//     set_intersection filters are restated line by line with hand-derivable known answers
//     (tests/test_oracle_normals.py, tests/test_oracle_downsample.py) and hashed into
//     tests/golden/oracle_golden.json.
// The Eigen-typed O(1) solves (JacobiSVD, LDLT, SelfAdjointEigenSolver) are "parity
// unpinned": Eigen3 is an external, unversioned dependency (CMakeLists.txt:7) absent here.
//
// ARITHMETIC CONTRACT (shared with the CUDA path; fp32, round-to-nearest, NO fma contraction —
// this file must be compiled with -ffp-contract=off):
//   sum3(a0,a1,a2)  = a0 + (a1 + a2)       Eigen redux_novec_unroller half-split of a 3-vector
//   q   = R s + t   : q_r = sum3(R_r0*x, R_r1*y, R_r2*z) + t_r
//                     correspondence_search/common_transformable_feature_adaptors.hpp:28-34
//   kNN d2          = ((dx*dx) + dy*dy) + dz*dz, d = q - ref     nanoflann.hpp:597-602 (tail loop)
//   k-means d2      = sum3(dx*dx, dy*dy, dz*dz), d = c - p       clustering/kmeans.hpp:108
//   RANSAC residual = sqrt(sum3(ex*ex, ey*ey, ez*ez)), e = (R s + t) - d
//                                                      model_estimation/ransac_transform_estimator.hpp:95
#include <cstdint>
#include <cstddef>
#include <cmath>
#include <cstring>
#include <limits>
#include <map>
#include <vector>
#include <random>
#include <algorithm>
#include <chrono>
#ifdef _OPENMP
#include <omp.h>
#endif
#include "small_linalg.hpp"

#define ORC_API extern "C" __attribute__((visibility("default")))

namespace {

inline float sum3(float a0, float a1, float a2) { return a0 + (a1 + a2); }

struct T34 {  // rigid transform, row-major [R | t], fp32 storage like Eigen::Transform<float,3,Isometry>
  float m[12];
  float R(int r, int c) const { return m[r * 4 + c]; }
  float t(int r) const { return m[r * 4 + 3]; }
};

inline T34 t34_identity() {
  T34 x;
  for (int i = 0; i < 12; i++) x.m[i] = 0.f;
  x.m[0] = x.m[5] = x.m[10] = 1.f;
  return x;
}

inline void apply(const T34& T, const float* s, float* q) {
  for (int r = 0; r < 3; r++) q[r] = sum3(T.R(r, 0) * s[0], T.R(r, 1) * s[1], T.R(r, 2) * s[2]) + T.t(r);
}

inline void rotate(const T34& T, const float* s, float* q) {
  for (int r = 0; r < 3; r++) q[r] = sum3(T.R(r, 0) * s[0], T.R(r, 1) * s[1], T.R(r, 2) * s[2]);
}

// a * b for rigid transforms; done in double and rounded once (Eigen does it in fp32 with an
// expression-template order we cannot pin; the difference is <= 1 ulp per entry).
inline T34 compose(const T34& a, const T34& b) {
  T34 r;
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) {
      double s = 0;
      for (int k = 0; k < 3; k++) s += (double)a.R(i, k) * (double)b.R(k, j);
      r.m[i * 4 + j] = (float)s;
    }
    double s = a.t(i);
    for (int k = 0; k < 3; k++) s += (double)a.R(i, k) * (double)b.t(k);
    r.m[i * 4 + 3] = (float)s;
  }
  return r;
}

struct Corr {  // core/correspondence.hpp:9-20
  size_t indexInFirst, indexInSecond;
  float value;
};

}  // namespace

// ---------------------------------------------------------------------------------------------
// Point transforms
// ---------------------------------------------------------------------------------------------

// PointFeaturesAdaptor::transformFeatures(tform) — common_transformable_feature_adaptors.hpp:28-34
// and transformPoints(tform, in, out) — core/space_transformations.hpp:203-216.
ORC_API void orc_transform_points(const float* T12, const float* src, size_t n, float* out) {
  T34 T;
  std::memcpy(T.m, T12, sizeof(T.m));
#pragma omp parallel for
  for (size_t i = 0; i < n; i++) apply(T, src + 3 * i, out + 3 * i);
}

// transformNormals for a rigid transform — core/space_transformations.hpp:374-390.
ORC_API void orc_rotate_vectors(const float* T12, const float* src, size_t n, float* out) {
  T34 T;
  std::memcpy(T.m, T12, sizeof(T.m));
#pragma omp parallel for
  for (size_t i = 0; i < n; i++) rotate(T, src + 3 * i, out + 3 * i);
}

// ---------------------------------------------------------------------------------------------
// 1-NN within a squared radius, brute force.
// Semantics of KDTree::kNNInRadiusSearch(q, k=1, r2) — core/kd_tree.hpp:284-291 with
// KNNSearchResultAdaptor (:63-109: slot pre-seeded with r2, replace only on strictly smaller)
// and the nanoflann leaf test `dist < worst_dist` (nanoflann.hpp:1901): the result is the
// reference point of minimum d2 provided d2 < r2; nothing otherwise. nanoflann breaks exact
// ties by traversal order; this brute-force form scans ascending index, so the LOWEST index
// wins a tie. idx = -1 and d2 = r2 when no neighbour qualifies.
// ---------------------------------------------------------------------------------------------
ORC_API void orc_knn1_brute(const float* ref, size_t nref, const float* qry, size_t nq, float max_d2,
                            int64_t* idx, float* d2) {
#pragma omp parallel for schedule(dynamic, 64)
  for (size_t i = 0; i < nq; i++) {
    const float qx = qry[3 * i], qy = qry[3 * i + 1], qz = qry[3 * i + 2];
    float best = max_d2;
    int64_t bi = -1;
    for (size_t j = 0; j < nref; j++) {
      const float dx = qx - ref[3 * j], dy = qy - ref[3 * j + 1], dz = qz - ref[3 * j + 2];
      float r = dx * dx;
      r = r + dy * dy;
      r = r + dz * dz;
      if (r < best) {
        best = r;
        bi = (int64_t)j;
      }
    }
    idx[i] = bi;
    d2[i] = best;
  }
}

// Unbounded 1-NN (KDTree::nearestNeighborSearch — core/kd_tree.hpp:181-193 → nanoflann
// KNNResultSet, nanoflann.hpp:196-282: initial worst = max float, strict `<`).
ORC_API void orc_nn1_brute(const float* ref, size_t nref, const float* qry, size_t nq, int64_t* idx,
                           float* d2) {
  orc_knn1_brute(ref, nref, qry, nq, std::numeric_limits<float>::max(), idx, d2);
}

// kNN search callback type: (user, transformed queries, nq, max_d2, idx out, d2 out).
// Either orc_knn1_brute_cb below or the nanoflann-backed one from oracle/_ref.
typedef void (*orc_knn_fn)(void* user, const float* qry, size_t nq, float max_d2, int64_t* idx, float* d2);

struct orc_brute_ctx {
  const float* ref;
  size_t nref;
};

ORC_API void orc_knn1_brute_cb(void* user, const float* qry, size_t nq, float max_d2, int64_t* idx,
                               float* d2) {
  const orc_brute_ctx* c = (const orc_brute_ctx*)user;
  orc_knn1_brute(c->ref, c->nref, qry, nq, max_d2, idx, d2);
}

// ---------------------------------------------------------------------------------------------
// findNNCorrespondencesUnidirectional, ref_is_first = true
// — correspondence_search/correspondence_search_kd_tree_utilities.hpp:7-51.
// keep[i] = found && evaluator(idx, i, d2) < max_distance (evaluator = identity,
// core/common_pair_evaluators.hpp:13-27); output compacted in query (src) order.
// ---------------------------------------------------------------------------------------------
static void find_correspondences(const float* qry_trans, size_t nq, size_t nref, float max_d2,
                                 orc_knn_fn knn, void* knn_user, std::vector<Corr>& out,
                                 std::vector<int64_t>& idx, std::vector<float>& d2) {
  out.clear();
  if (nref == 0) return;  // :16-19
  idx.resize(nq);
  d2.resize(nq);
  knn(knn_user, qry_trans, nq, max_d2, idx.data(), d2.data());
  out.reserve(nq);
  for (size_t i = 0; i < nq; i++) {
    if (idx[i] >= 0 && d2[i] < max_d2) out.push_back({(size_t)idx[i], i, d2[i]});
  }
}

ORC_API size_t orc_find_correspondences(const float* T12, const float* src, size_t nsrc, size_t nref,
                                        float max_d2, orc_knn_fn knn, void* knn_user,
                                        uint64_t* idx_first, uint64_t* idx_second, float* value) {
  std::vector<float> q(3 * nsrc);
  orc_transform_points(T12, src, nsrc, q.data());
  std::vector<Corr> corr;
  std::vector<int64_t> idx;
  std::vector<float> d2;
  find_correspondences(q.data(), nsrc, nref, max_d2, knn, knn_user, corr, idx, d2);
  for (size_t i = 0; i < corr.size(); i++) {
    idx_first[i] = corr[i].indexInFirst;
    idx_second[i] = corr[i].indexInSecond;
    value[i] = corr[i].value;
  }
  return corr.size();
}

// ---------------------------------------------------------------------------------------------
// LinearTransform::rotation() — core/space_transformations.hpp:43-51
// ---------------------------------------------------------------------------------------------
static void reorthonormalize(T34& T) {
  orc::M3 A;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) A.a[i][j] = T.R(i, j);
  orc::M3 R = orc::nearest_rotation_col0_rule(A);
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) T.m[i * 4 + j] = (float)R.a[i][j];
}

ORC_API void orc_rotation(const float* L9_rowmajor, float* out9_rowmajor) {
  orc::M3 A;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) A.a[i][j] = L9_rowmajor[i * 3 + j];
  orc::M3 R = orc::nearest_rotation_col0_rule(A);
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) out9_rowmajor[i * 3 + j] = (float)R.a[i][j];
}

// ---------------------------------------------------------------------------------------------
// estimateTransformPointToPointMetric, rigid — registration/transform_estimation.hpp:12-48.
// dst/src are already-corresponding packed xyz sets of equal length n. Accumulations are fp32
// in serial order (the ENABLE_NON_DETERMINISTIC_PARALLELISM=OFF build); `accum_double` switches
// the three O(n) sums to double (used to bound the reference's own fp32 accumulation noise).
// ---------------------------------------------------------------------------------------------
template <typename Acc>
static bool kabsch(const float* dst, const float* src, size_t n, T34& tform) {
  if (n == 0) {  // :20-23
    tform = t34_identity();
    return false;
  }
  // :25-26  rowwise().mean(): serial sum of each row, divided by the count
  Acc sd[3] = {0, 0, 0}, ss[3] = {0, 0, 0};
  for (size_t i = 0; i < n; i++)
    for (int r = 0; r < 3; r++) {
      sd[r] += (Acc)dst[3 * i + r];
      ss[r] += (Acc)src[3 * i + r];
    }
  float mu_d[3], mu_s[3];
  for (int r = 0; r < 3; r++) {
    mu_d[r] = (float)(sd[r] / (Acc)n);
    mu_s[r] = (float)(ss[r] / (Acc)n);
  }
  // :28-34  sigma = (1/n) * (dst - mu_d) (src - mu_s)^T
  Acc sig[3][3] = {{0}};
  for (size_t i = 0; i < n; i++) {
    float dc[3], sc[3];
    for (int r = 0; r < 3; r++) {
      dc[r] = dst[3 * i + r] - mu_d[r];
      sc[r] = src[3 * i + r] - mu_s[r];
    }
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) sig[r][c] += (Acc)(dc[r] * sc[c]);
  }
  orc::M3 S;
  const float inv_n = 1.0f / (float)n;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) S.a[r][c] = (float)(inv_n * (float)sig[r][c]);
  // :36-44
  orc::M3 R = orc::kabsch_rotation_from_sigma(S);
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) tform.m[r * 4 + c] = (float)R.a[r][c];
  // :45  t = mu_dst - R * mu_src
  for (int r = 0; r < 3; r++)
    tform.m[r * 4 + 3] = mu_d[r] - sum3(tform.R(r, 0) * mu_s[0], tform.R(r, 1) * mu_s[1], tform.R(r, 2) * mu_s[2]);
  return n >= 3;  // :47
}

ORC_API int orc_kabsch(const float* dst, const float* src, size_t n, int accum_double, float* T12) {
  T34 T;
  bool ok = accum_double ? kabsch<double>(dst, src, n, T) : kabsch<float>(dst, src, n, T);
  std::memcpy(T12, T.m, sizeof(T.m));
  return ok ? 1 : 0;
}

// corr overload — transform_estimation.hpp:104-113 + selectCorrespondingPoints correspondence.hpp:146-159
template <typename Acc>
static bool kabsch_corr(const float* dst, const float* src, const std::vector<Corr>& corr, T34& tform) {
  std::vector<float> d(3 * corr.size()), s(3 * corr.size());
  for (size_t i = 0; i < corr.size(); i++)
    for (int r = 0; r < 3; r++) {
      d[3 * i + r] = dst[3 * corr[i].indexInFirst + r];
      s[3 * i + r] = src[3 * corr[i].indexInSecond + r];
    }
  return kabsch<Acc>(d.data(), s.data(), corr.size(), tform);
}

// ---------------------------------------------------------------------------------------------
// estimateTransformCombinedMetric rigid 3-D — transform_estimation.hpp:238-367, and
// estimateTransformSymmetricMetric — :608-739 (src_n != nullptr; n = n_dst + R_tform n_src).
// Correspondence weight evaluators: UnityWeightEvaluator (common_pair_evaluators.hpp:29-43) => weight = metric
// weight; RBFKernelWeightEvaluator<float, float, true> (:46-79) => metric weight * std::exp(coeff_ * value) with
// coeff_ = -(0.5f) / (sigma * sigma), value = the correspondence's squared distance (called as
// evaluator(indexInFirst, indexInSecond, value), transform_estimation.hpp:302-304 / :331-333).
// ---------------------------------------------------------------------------------------------
struct CorrWeights {
  int pt_kind = 0, pl_kind = 0;  // 0 unity, 1 RBF
  float pt_coeff = -0.5f, pl_coeff = -0.5f;
};
static inline float corr_weight(int kind, float coeff, float value) { return kind ? std::exp(coeff * value) : 1.f; }

template <typename Acc>
static void accumulate_combined(const float* dst_p, const float* dst_n, const float* src_p, const float* src_n,
                                const Corr* corr, size_t begin, size_t end, bool has_pt, bool has_pl,
                                float w_pt_metric, float w_pl_metric, const T34& tform, const float* dst_mean,
                                const float* src_mean, Acc AtA[36], Acc Atb[6], const CorrWeights& cw = CorrWeights()) {
  if (has_pt) {  // :292-321
    for (size_t i = begin; i < end; i++) {
      const Corr& c = corr[i];
      const float w_pt = w_pt_metric * corr_weight(cw.pt_kind, cw.pt_coeff, c.value);  // :302-304
      float d[3], sm[3], s[3];
      for (int r = 0; r < 3; r++) d[r] = dst_p[3 * c.indexInFirst + r] - dst_mean[r];
      for (int r = 0; r < 3; r++) sm[r] = src_p[3 * c.indexInSecond + r] - src_mean[r];
      apply(tform, sm, s);
      float E[6][3];
      E[0][0] = 0.f; E[1][1] = 0.f; E[2][2] = 0.f;
      E[0][1] = -(d[2] + s[2]);
      E[0][2] = (d[1] + s[1]);
      E[1][2] = -(d[0] + s[0]);
      E[1][0] = -E[0][1];
      E[2][0] = -E[0][2];
      E[2][1] = -E[1][2];
      for (int r = 0; r < 3; r++)
        for (int cc = 0; cc < 3; cc++) E[3 + r][cc] = (r == cc) ? 1.f : 0.f;
      float ds[3] = {d[0] - s[0], d[1] - s[1], d[2] - s[2]};
      for (int r = 0; r < 6; r++) {
        for (int cc = 0; cc < 6; cc++) {
          float v = sum3(E[r][0] * E[cc][0], E[r][1] * E[cc][1], E[r][2] * E[cc][2]);
          AtA[r * 6 + cc] += (Acc)(w_pt * v);
        }
        Atb[r] += (Acc)(w_pt * sum3(E[r][0] * ds[0], E[r][1] * ds[1], E[r][2] * ds[2]));
      }
    }
  }
  if (has_pl) {  // :323-343 / :694-715
    for (size_t i = begin; i < end; i++) {
      const Corr& c = corr[i];
      const float w_pl = w_pl_metric * corr_weight(cw.pl_kind, cw.pl_coeff, c.value);  // :331-333
      float d[3], n[3], sm[3], s[3];
      for (int r = 0; r < 3; r++) d[r] = dst_p[3 * c.indexInFirst + r] - dst_mean[r];
      for (int r = 0; r < 3; r++) n[r] = dst_n[3 * c.indexInFirst + r];
      if (src_n) {  // :705-706
        float rn[3];
        rotate(tform, src_n + 3 * c.indexInSecond, rn);
        for (int r = 0; r < 3; r++) n[r] = n[r] + rn[r];
      }
      for (int r = 0; r < 3; r++) sm[r] = src_p[3 * c.indexInSecond + r] - src_mean[r];
      apply(tform, sm, s);
      float v[3] = {d[0] + s[0], d[1] + s[1], d[2] + s[2]};
      float a[6];
      a[0] = v[1] * n[2] - v[2] * n[1];
      a[1] = v[2] * n[0] - v[0] * n[2];
      a[2] = v[0] * n[1] - v[1] * n[0];
      a[3] = n[0]; a[4] = n[1]; a[5] = n[2];
      float ds[3] = {d[0] - s[0], d[1] - s[1], d[2] - s[2]};
      float ndot = sum3(n[0] * ds[0], n[1] * ds[1], n[2] * ds[2]);
      for (int r = 0; r < 6; r++) {
        for (int cc = 0; cc < 6; cc++) AtA[r * 6 + cc] += (Acc)((w_pl * a[r]) * a[cc]);
        Atb[r] += (Acc)((w_pl * ndot) * a[r]);
      }
    }
  }
}

template <typename Acc>
static bool estimate_combined(const float* dst_p, const float* dst_n, size_t n_dst_p, size_t n_dst_n,
                              const float* src_p, const float* src_n, const std::vector<Corr>& corr,
                              float w_pt, float w_pl, size_t max_iter, float tol, const float* dst_mean,
                              const float* src_mean, bool parallel, T34& tform, const CorrWeights& cw = CorrWeights()) {
  tform = t34_identity();  // :262
  const bool has_pt = !corr.empty() && (w_pt > 0.f);
  const bool has_pl = !corr.empty() && (w_pl > 0.f);
  if ((!has_pt && !has_pl) || (has_pl && n_dst_p != n_dst_n)) return false;  // :269-272

  for (size_t iter = 0; iter < max_iter; ++iter) {
    Acc AtA[36], Atb[6];
    for (int i = 0; i < 36; i++) AtA[i] = 0;
    for (int i = 0; i < 6; i++) Atb[i] = 0;
    if (!parallel) {
      accumulate_combined<Acc>(dst_p, dst_n, src_p, src_n, corr.data(), 0, corr.size(), has_pt, has_pl, w_pt,
                               w_pl, tform, dst_mean, src_mean, AtA, Atb, cw);
    } else {
      // ENABLE_NON_DETERMINISTIC_PARALLELISM=ON build (:285-290): per-thread partials, summed.
#ifdef _OPENMP
      int nt = omp_get_max_threads();
#else
      int nt = 1;
#endif
      std::vector<Acc> part((size_t)nt * 42, (Acc)0);
#pragma omp parallel num_threads(nt)
      {
#ifdef _OPENMP
        int t = omp_get_thread_num();
#else
        int t = 0;
#endif
        size_t chunk = (corr.size() + nt - 1) / nt;
        size_t b = std::min(corr.size(), chunk * t), e = std::min(corr.size(), b + chunk);
        accumulate_combined<Acc>(dst_p, dst_n, src_p, src_n, corr.data(), b, e, has_pt, has_pl, w_pt, w_pl,
                                 tform, dst_mean, src_mean, &part[(size_t)t * 42], &part[(size_t)t * 42 + 36], cw);
      }
      for (int t = 0; t < nt; t++) {
        for (int i = 0; i < 36; i++) AtA[i] += part[(size_t)t * 42 + i];
        for (int i = 0; i < 6; i++) Atb[i] += part[(size_t)t * 42 + 36 + i];
      }
    }
    // :346  d_theta = AtA.ldlt().solve(Atb)   (fp32 system as the reference holds it, solved in double)
    double A[36], b[6], x[6];
    for (int i = 0; i < 36; i++) A[i] = (double)(float)AtA[i];
    for (int i = 0; i < 6; i++) b[i] = (double)(float)Atb[i];
    orc::ldlt6_solve(A, b, x);
    float dth[6];
    for (int i = 0; i < 6; i++) dth[i] = (float)x[i];

    // :349-357  Ra = AngleAxis(atan(|w|), w/|w|), ta = cos(theta) * d_theta.tail<3>,
    //           tform = Ra * ta * Ra * tform
    double na = std::sqrt((double)dth[0] * dth[0] + (double)dth[1] * dth[1] + (double)dth[2] * dth[2]);
    double theta = std::atan(na);
    double ax[3] = {0, 0, 0};
    if (na > 0) {
      ax[0] = dth[0] / na; ax[1] = dth[1] / na; ax[2] = dth[2] / na;
    }
    double cth = std::cos(theta), sth = std::sin(theta), omc = 1.0 - cth;
    orc::M3 Ra;
    Ra.a[0][0] = cth + omc * ax[0] * ax[0];
    Ra.a[0][1] = omc * ax[0] * ax[1] - sth * ax[2];
    Ra.a[0][2] = omc * ax[0] * ax[2] + sth * ax[1];
    Ra.a[1][0] = omc * ax[1] * ax[0] + sth * ax[2];
    Ra.a[1][1] = cth + omc * ax[1] * ax[1];
    Ra.a[1][2] = omc * ax[1] * ax[2] - sth * ax[0];
    Ra.a[2][0] = omc * ax[2] * ax[0] - sth * ax[1];
    Ra.a[2][1] = omc * ax[2] * ax[1] + sth * ax[0];
    Ra.a[2][2] = cth + omc * ax[2] * ax[2];
    double ta[3] = {cth * dth[3], cth * dth[4], cth * dth[5]};
    // M = Ra * Translate(ta) * Ra * tform  ->  linear = Ra Ra L ; trans = Ra (Ra t + ta)
    orc::M3 L;
    double t0[3];
    for (int i = 0; i < 3; i++) {
      for (int j = 0; j < 3; j++) L.a[i][j] = tform.R(i, j);
      t0[i] = tform.t(i);
    }
    orc::M3 RL = orc::m3_mul(Ra, L);
    double t1[3], t2[3];
    for (int i = 0; i < 3; i++) t1[i] = Ra.a[i][0] * t0[0] + Ra.a[i][1] * t0[1] + Ra.a[i][2] * t0[2] + ta[i];
    for (int i = 0; i < 3; i++) t2[i] = Ra.a[i][0] * t1[0] + Ra.a[i][1] * t1[1] + Ra.a[i][2] * t1[2];
    orc::M3 RRL = orc::m3_mul(Ra, RL);
    for (int i = 0; i < 3; i++) {
      for (int j = 0; j < 3; j++) tform.m[i * 4 + j] = (float)RRL.a[i][j];
      tform.m[i * 4 + 3] = (float)t2[i];
    }
    // :360-363
    double nrm = 0;
    for (int i = 0; i < 6; i++) nrm += (double)dth[i] * dth[i];
    bool conv = (float)std::sqrt(nrm) < tol;
    if (conv || iter + 1 == max_iter) {
      // :361/:365  tform = Translation(dst_mean) * tform * Translation(-src_mean)
      for (int i = 0; i < 3; i++) {
        double tt = tform.t(i);
        for (int k = 0; k < 3; k++) tt -= (double)tform.R(i, k) * (double)src_mean[k];
        tform.m[i * 4 + 3] = (float)(tt + (double)dst_mean[i]);
      }
      return conv;
    }
  }
  // max_iter == 0: :365 still applies the un-centring to the identity
  for (int i = 0; i < 3; i++) tform.m[i * 4 + 3] = (float)((double)dst_mean[i] - (double)src_mean[i]);
  return false;
}

ORC_API int orc_estimate_combined(const float* dst_p, const float* dst_n, size_t n_dst, const float* src_p,
                                  const float* src_n_or_null, const uint64_t* idx_first,
                                  const uint64_t* idx_second, size_t n_corr, float w_pt, float w_pl,
                                  size_t max_iter, float tol, const float* dst_mean, const float* src_mean,
                                  int accum_double, float* T12) {
  std::vector<Corr> corr(n_corr);
  for (size_t i = 0; i < n_corr; i++) corr[i] = {(size_t)idx_first[i], (size_t)idx_second[i], 0.f};
  T34 T;
  bool ok = accum_double
                ? estimate_combined<double>(dst_p, dst_n, n_dst, n_dst, src_p, src_n_or_null, corr, w_pt, w_pl,
                                            max_iter, tol, dst_mean, src_mean, false, T)
                : estimate_combined<float>(dst_p, dst_n, n_dst, n_dst, src_p, src_n_or_null, corr, w_pt, w_pl,
                                           max_iter, tol, dst_mean, src_mean, false, T);
  std::memcpy(T12, T.m, sizeof(T.m));
  return ok ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------
// ICP drivers.
//   IterativeClosestPointBase::estimate()                      registration/icp_base.hpp:68-87
//   PointToPointMetricSingleTransformICP::updateEstimate()     icp_single_transform_point_to_point_metric.hpp:46-65
//   CombinedMetricSingleTransformICP ctor means / updateEstimate()
//                                                              icp_single_transform_combined_metric.hpp:51-58,173-217
//   CorrespondenceSearchKDTree::findCorrespondences(tform)     correspondence_search_kd_tree.hpp:185-229
//     (defaults SECOND_TO_FIRST, inlier_fraction 1, no reciprocity / one-to-one, :49-51)
// ---------------------------------------------------------------------------------------------
struct orc_icp_params {
  int32_t metric;        // 0 = point-to-point (Kabsch), 1 = combined / symmetric Gauss-Newton
  int32_t max_iter;      // icp_base.hpp:24 (default 15)
  float tol;             // icp_base.hpp:25 (default 1e-5)
  float max_d2;          // SQUARED max correspondence distance (correspondence_search_kd_tree.hpp:49, 1e-4)
  float w_pt, w_pl;      // combined: defaults 0, 1 (icp_single_transform_combined_metric.hpp:46-47)
  int32_t max_opt_iter;  // default 1 (:44)
  float opt_tol;         // default 1e-5 (:45)
  int32_t accum_double;  // 0 = faithful fp32 accumulation, 1 = double accumulation
  int32_t parallel;      // 1 = ENABLE_NON_DETERMINISTIC_PARALLELISM-style OpenMP reduction (timing runs)
  float T_init[12];      // icp_base.hpp:58-61
  // correspondence-engine options (correspondence_search_kd_tree.hpp:46-50); defaults 0, 0, 0, 1.0
  int32_t search_dir;          // 0 SECOND_TO_FIRST, 1 FIRST_TO_SECOND, 2 BOTH
  int32_t require_reciprocal;
  int32_t one_to_one;
  int32_t reserved_;
  double inlier_fraction;
  // FIRST_TO_SECOND / BOTH: 1-NN of the dst points among the transformed src points, tree rebuilt per call.
  // nullptr = orc_knn1_brute; tests pass oracle/_ref's ref_knn1_build_query (the reference's own nanoflann).
  void (*f2s_fn)(const float* ref_pts, size_t nref, const float* qry, size_t nq, float max_d2, int64_t* idx, float* d2);
  // correspondence weight evaluators of the combined metric: 0 = UnityWeightEvaluator, 1 = RBFKernelWeightEvaluator
  int32_t pt_weight_kind, pl_weight_kind;
  float pt_weight_coeff, pl_weight_coeff;  // -(0.5f) / (sigma * sigma)
};

// CorrespondenceSearchKDTree::findCorrespondences(tform) — correspondence_search_kd_tree.hpp:107-229:
//   SECOND_TO_FIRST (:205-213)  queries = transformed src against the dst tree (the knn callback)
//   FIRST_TO_SECOND (:195-204)  queries = dst against a tree over the transformed src, rebuilt per call —
//                               restated by brute force (orc_knn1_brute: same distance arithmetic, lowest
//                               index on exact ties); small inputs only
//   BOTH (:214-226)             both lists sorted lexicographically on (first, second), then set_union, or
//                               set_intersection when require_reciprocal
//                               (correspondence_search_kd_tree_utilities.hpp:64-99)
//   filterCorrespondencesFraction (core/correspondence.hpp:57-66): sort by value, keep llround(f * size)
//   filterCorrespondencesOneToOne (:68-100): sort by (index, value), keep the first pair per index
// std::sort leaves equal keys in unspecified order; stable_sort pins the rule shared with the CUDA path:
// ties keep the order of the list the filter received.
static void engine_correspondences(const float* dst_p, size_t n_dst, const float* src_trans, size_t n_src,
                                   const orc_icp_params* prm, orc_knn_fn knn, void* knn_user,
                                   std::vector<Corr>& corr, std::vector<int64_t>& idx, std::vector<float>& d2) {
  std::vector<Corr> s2f, f2s;
  const int dir = prm->search_dir;
  if (dir != 1) find_correspondences(src_trans, n_src, n_dst, prm->max_d2, knn, knn_user, s2f, idx, d2);
  if (dir != 0 && n_src > 0 && n_dst > 0) {
    std::vector<int64_t> j(n_dst);
    std::vector<float> v(n_dst);
    (prm->f2s_fn ? prm->f2s_fn : orc_knn1_brute)(src_trans, n_src, dst_p, n_dst, prm->max_d2, j.data(), v.data());
    for (size_t i = 0; i < n_dst; i++)
      if (j[i] >= 0 && v[i] < prm->max_d2) f2s.push_back({i, (size_t)j[i], v[i]});
  }
  auto lex = [](const Corr& a, const Corr& b) {
    return a.indexInFirst != b.indexInFirst ? a.indexInFirst < b.indexInFirst : a.indexInSecond < b.indexInSecond;
  };
  corr.clear();
  if (dir == 0) {
    corr = s2f;
  } else if (dir == 1) {
    corr = f2s;
  } else {
    std::sort(f2s.begin(), f2s.end(), lex);
    std::sort(s2f.begin(), s2f.end(), lex);
    if (prm->require_reciprocal)
      std::set_intersection(f2s.begin(), f2s.end(), s2f.begin(), s2f.end(), std::back_inserter(corr), lex);
    else
      std::set_union(f2s.begin(), f2s.end(), s2f.begin(), s2f.end(), std::back_inserter(corr), lex);
  }
  const double f = prm->inlier_fraction;
  if (f > 0.0 && f < 1.0) {
    std::stable_sort(corr.begin(), corr.end(), [](const Corr& a, const Corr& b) { return a.value < b.value; });
    corr.erase(corr.begin() + std::llround(f * (double)corr.size()), corr.end());
  }
  if (prm->one_to_one && !corr.empty() && dir != 2) {
    std::vector<Corr> copy = corr;
    corr.clear();
    if (dir == 1) {
      std::stable_sort(copy.begin(), copy.end(), [](const Corr& a, const Corr& b) {
        return a.indexInSecond != b.indexInSecond ? a.indexInSecond < b.indexInSecond : a.value < b.value;
      });
      corr.push_back(copy.front());
      for (const Corr& c : copy)
        if (c.indexInSecond != corr.back().indexInSecond) corr.push_back(c);
    } else {
      std::stable_sort(copy.begin(), copy.end(), [](const Corr& a, const Corr& b) {
        return a.indexInFirst != b.indexInFirst ? a.indexInFirst < b.indexInFirst : a.value < b.value;
      });
      corr.push_back(copy.front());
      for (const Corr& c : copy)
        if (c.indexInFirst != corr.back().indexInFirst) corr.push_back(c);
    }
  }
}

static bool engine_mode(const orc_icp_params* p) {
  return p->search_dir != 0 || p->one_to_one != 0 || (p->inlier_fraction > 0.0 && p->inlier_fraction < 1.0);
}

struct orc_icp_result {
  float T[12];
  int32_t iterations;
  float last_delta;
  int32_t converged;
  uint64_t last_num_corr;
  double t_knn_s, t_est_s;  // wall-clock split (for the CPU baseline)
};

static void colmean(const float* p, size_t n, float* mu) {
  // rowwise().mean() of a 3 x n column-major map: serial fp32 sum per row, / n
  float s[3] = {0, 0, 0};
  for (size_t i = 0; i < n; i++)
    for (int r = 0; r < 3; r++) s[r] += p[3 * i + r];
  for (int r = 0; r < 3; r++) mu[r] = (n == 0) ? 0.f : s[r] / (float)n;
}

ORC_API void orc_icp(const float* dst_p, const float* dst_n, size_t n_dst, const float* src_p,
                     const float* src_n, size_t n_src, const orc_icp_params* prm, orc_knn_fn knn,
                     void* knn_user, orc_icp_result* res, float* T_log /* max_iter*12 or null */) {
  using clk = std::chrono::steady_clock;
  T34 T;
  std::memcpy(T.m, prm->T_init, sizeof(T.m));  // icp_base.hpp:71
  float dst_mean[3] = {0, 0, 0}, src_mean[3] = {0, 0, 0};
  if (prm->metric == 1) {
    colmean(dst_p, n_dst, dst_mean);
    colmean(src_p, n_src, src_mean);
  }
  std::vector<float> src_trans(3 * n_src), src_n_trans;
  if (src_n) src_n_trans.resize(3 * n_src);
  std::vector<Corr> corr;
  std::vector<int64_t> idx;
  std::vector<float> d2;
  int iters = 0;
  float last_delta = std::numeric_limits<float>::infinity();
  double t_knn = 0, t_est = 0;
  while (iters < prm->max_iter) {
    auto t0 = clk::now();
    // updateCorrespondences(): transformFeatures(T) then the radius-bounded 1-NN sweep
    orc_transform_points(T.m, src_p, n_src, src_trans.data());
    if (engine_mode(prm))
      engine_correspondences(dst_p, n_dst, src_trans.data(), n_src, prm, knn, knn_user, corr, idx, d2);
    else
      find_correspondences(src_trans.data(), n_src, n_dst, prm->max_d2, knn, knn_user, corr, idx, d2);
    auto t1 = clk::now();
    // updateEstimate(): transformPoints(T, src) again (same values), then the estimator
    T34 Titer;
    if (prm->metric == 0) {
      if (prm->accum_double)
        kabsch_corr<double>(dst_p, src_trans.data(), corr, Titer);
      else
        kabsch_corr<float>(dst_p, src_trans.data(), corr, Titer);
    } else {
      float src_mean_t[3];
      apply(T, src_mean, src_mean_t);  // this->transform_ * src_mean_  (:189/:196)
      const float* sn = nullptr;
      if (src_n) {
        orc_rotate_vectors(T.m, src_n, n_src, src_n_trans.data());  // transformNormals :183
        sn = src_n_trans.data();
      }
      CorrWeights cw;
      cw.pt_kind = prm->pt_weight_kind;
      cw.pl_kind = prm->pl_weight_kind;
      cw.pt_coeff = prm->pt_weight_coeff;
      cw.pl_coeff = prm->pl_weight_coeff;
      if (prm->accum_double)
        estimate_combined<double>(dst_p, dst_n, n_dst, n_dst, src_trans.data(), sn, corr, prm->w_pt, prm->w_pl,
                                  (size_t)prm->max_opt_iter, prm->opt_tol, dst_mean, src_mean_t,
                                  prm->parallel != 0, Titer, cw);
      else
        estimate_combined<float>(dst_p, dst_n, n_dst, n_dst, src_trans.data(), sn, corr, prm->w_pt, prm->w_pl,
                                 (size_t)prm->max_opt_iter, prm->opt_tol, dst_mean, src_mean_t,
                                 prm->parallel != 0, Titer, cw);
    }
    reorthonormalize(Titer);  // :207-211 / p2p :56-60
    T = compose(Titer, T);    // :213
    float dn = 0.f;           // :214-216
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) {
        float e = Titer.R(r, c) - (r == c ? 1.f : 0.f);
        dn += e * e;
      }
      dn += Titer.t(r) * Titer.t(r);
    }
    last_delta = std::sqrt(dn);
    auto t2 = clk::now();
    t_knn += std::chrono::duration<double>(t1 - t0).count();
    t_est += std::chrono::duration<double>(t2 - t1).count();
    if (T_log) std::memcpy(T_log + 12 * iters, T.m, sizeof(T.m));
    iters++;
    if (last_delta < prm->tol) break;  // icp_base.hpp:83
  }
  std::memcpy(res->T, T.m, sizeof(T.m));
  res->iterations = iters;
  res->last_delta = last_delta;
  res->converged = last_delta < prm->tol;
  res->last_num_corr = corr.size();
  res->t_knn_s = t_knn;
  res->t_est_s = t_est;
}

// getCorrespondences() after findCorrespondences(T) with the engine options of prm (tests).
ORC_API size_t orc_engine_correspondences(const float* dst_p, size_t n_dst, const float* src_p, size_t n_src,
                                          const float* T12, const orc_icp_params* prm, orc_knn_fn knn,
                                          void* knn_user, uint64_t* idx_first, uint64_t* idx_second, float* value) {
  std::vector<float> q(3 * n_src);
  orc_transform_points(T12, src_p, n_src, q.data());
  std::vector<Corr> corr;
  std::vector<int64_t> idx;
  std::vector<float> d2;
  engine_correspondences(dst_p, n_dst, q.data(), n_src, prm, knn, knn_user, corr, idx, d2);
  for (size_t i = 0; i < corr.size(); i++) {
    idx_first[i] = corr[i].indexInFirst;
    idx_second[i] = corr[i].indexInSecond;
    value[i] = corr[i].value;
  }
  return corr.size();
}

// computeResiduals() — icp_single_transform_combined_metric.hpp:220-243 (metric 1) and
// icp_single_transform_point_to_point_metric.hpp:68-85 (metric 0): unbounded 1-NN of T*src_i,
// res_i = w_pt |d - q|^2 + w_pl (n . (d - q))^2 ; NaN-filled when dst is empty.
ORC_API void orc_icp_residuals(const float* dst_p, const float* dst_n, size_t n_dst, const float* src_p,
                               const float* src_n, size_t n_src, const float* T12, int metric, float w_pt,
                               float w_pl, orc_knn_fn knn, void* knn_user, float* res) {
  if (n_dst == 0) {
    for (size_t i = 0; i < n_src; i++) res[i] = std::numeric_limits<float>::quiet_NaN();
    return;
  }
  std::vector<float> q(3 * n_src), d2(n_src);
  std::vector<int64_t> idx(n_src);
  orc_transform_points(T12, src_p, n_src, q.data());
  knn(knn_user, q.data(), n_src, std::numeric_limits<float>::max(), idx.data(), d2.data());
  for (size_t i = 0; i < n_src; i++) {
    const float* d = dst_p + 3 * idx[i];
    float e[3] = {d[0] - q[3 * i], d[1] - q[3 * i + 1], d[2] - q[3 * i + 2]};
    float sq = sum3(e[0] * e[0], e[1] * e[1], e[2] * e[2]);
    if (metric == 0) {
      res[i] = sq;
    } else {
      float n[3] = {dst_n[3 * idx[i]], dst_n[3 * idx[i] + 1], dst_n[3 * idx[i] + 2]};
      if (src_n)
        for (int r = 0; r < 3; r++) n[r] += src_n[3 * i + r];  // :236 (un-rotated, as the reference does)
      float pd = sum3(n[0] * e[0], n[1] * e[1], n[2] * e[2]);
      res[i] = w_pt * sq + w_pl * pd * pd;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// KMeans::cluster_ — clustering/kmeans.hpp:67-194 (brute-force assignment branch :96-119).
// ---------------------------------------------------------------------------------------------
static inline float kmeans_d2(const float* c, const float* p) {
  float dx = c[0] - p[0], dy = c[1] - p[1], dz = c[2] - p[2];
  return sum3(dx * dx, dy * dy, dz * dz);
}

// One assignment sweep (:100-119). Returns 1 if no label changed.
ORC_API int orc_kmeans_assign(const float* pts, size_t n, const float* cent, size_t k, uint64_t* labels) {
  int unchanged = 1;
#pragma omp parallel for schedule(static) reduction(&& : unchanged)
  for (size_t i = 0; i < n; i++) {
    float min_dist = std::numeric_limits<float>::infinity();
    uint64_t min_ind = 0;
    for (size_t j = 0; j < k; j++) {
      float d = kmeans_d2(cent + 3 * j, pts + 3 * i);
      if (d < min_dist) {
        min_dist = d;
        min_ind = j;
      }
    }
    if (labels[i] != min_ind) unchanged = 0;
    labels[i] = min_ind;
  }
  return unchanged;
}

// cluster(num_clusters, ...) seeding — kmeans.hpp:32-49, with the seed injected in place of
// std::random_device (SURVEY.md F8).
ORC_API void orc_kmeans_seed_indices(size_t n, size_t k, uint32_t seed, uint64_t* out_idx) {
  std::vector<size_t> range(n);
  for (size_t i = 0; i < n; i++) range[i] = i;
  std::mt19937 rng(seed);
  size_t prev = n;
  for (size_t i = 0; i < k; i++) {
    std::uniform_int_distribution<size_t> dist(0, prev - 1);
    size_t r = dist(rng);
    out_idx[i] = range[r];
    prev--;
    std::swap(range[r], range[prev]);
  }
}

// Full Lloyd loop. centroids: in = initial, out = final (k x 3 packed). labels: n (zero-filled on entry
// like the freshly resized point_to_cluster_index_map_, :82). Returns performed iterations.
ORC_API size_t orc_kmeans(const float* pts, size_t n, float* cent, size_t k, size_t max_iter, float tol,
                          uint64_t* labels) {
  const float tol_sq = tol * tol;
  std::vector<float> old;
  for (size_t i = 0; i < n; i++) labels[i] = 0;
  size_t it = 0;
  while (it < max_iter) {
    int unchanged = orc_kmeans_assign(pts, n, cent, k, labels);
    if (unchanged && it > 0) break;                  // :122
    if (tol > 0.f) old.assign(cent, cent + 3 * k);   // :123
    // :126-131  serial fp32 accumulation
    for (size_t j = 0; j < 3 * k; j++) cent[j] = 0.f;
    std::vector<size_t> cnt(k, 0);
    for (size_t i = 0; i < n; i++) {
      float* c = cent + 3 * labels[i];
      c[0] += pts[3 * i];
      c[1] += pts[3 * i + 1];
      c[2] += pts[3 * i + 2];
      cnt[labels[i]]++;
    }
    // :134-176  empty-cluster repair
    for (size_t i = 0; i < k; i++) {
      if (cnt[i] != 0) continue;
      size_t max_ind = 0;
      for (size_t j = 1; j < k; j++)
        if (cnt[j] > cnt[max_ind]) max_ind = j;
      float inv = 1.0f / (float)cnt[max_ind];
      float oc[3] = {cent[3 * max_ind] * inv, cent[3 * max_ind + 1] * inv, cent[3 * max_ind + 2] * inv};
      float max_dist = -1.0f;
      size_t max_dist_ind = 0;
      for (size_t j = 0; j < n; j++) {  // serial: first maximal element wins (the omp critical
        if (labels[j] == max_ind) {     // version is order-dependent only on exact ties)
          float d = kmeans_d2(oc, pts + 3 * j);
          if (d > max_dist) {
            max_dist = d;
            max_dist_ind = j;
          }
        }
      }
      labels[max_dist_ind] = i;
      for (int r = 0; r < 3; r++) cent[3 * max_ind + r] -= pts[3 * max_dist_ind + r];
      cnt[max_ind]--;
      cnt[i]++;
      // NB (:172-175): the moved point is NOT added to centroid i's sum; it stays 0 * (1/1).
    }
    for (size_t i = 0; i < k; i++) {  // :179-181
      float inv = 1.0f / (float)cnt[i];
      for (int r = 0; r < 3; r++) cent[3 * i + r] *= inv;
    }
    it++;
    if (tol > 0.f) {  // :186-188
      float mx = 0.f;
      for (size_t i = 0; i < k; i++) mx = std::max(mx, kmeans_d2(cent + 3 * i, old.data() + 3 * i));
      if (mx < tol_sq) break;
    }
  }
  return it;
}

// ---------------------------------------------------------------------------------------------
// RANSAC — model_estimation/ransac_base.hpp:64-131 with
// TransformRANSACEstimator<RigidTransform3f> — ransac_transform_estimator.hpp:72-98.
// ---------------------------------------------------------------------------------------------
static inline float ransac_residual(const T34& T, const float* s, const float* d) {
  float q[3];
  apply(T, s, q);
  float e[3] = {q[0] - d[0], q[1] - d[1], q[2] - d[2]};
  return std::sqrt(sum3(e[0] * e[0], e[1] * e[1], e[2] * e[2]));
}

// computeResiduals + the serial `<= thresh` scan (ransac_transform_estimator.hpp:90-98,
// ransac_base.hpp:96-101) for H hypotheses given as row-major [R|t] 3x4 blocks.
ORC_API void orc_ransac_score(const float* dst, const float* src, size_t n, const float* T_h, size_t H,
                              float thresh, uint32_t* counts) {
#pragma omp parallel for schedule(dynamic, 1)
  for (size_t h = 0; h < H; h++) {
    T34 T;
    std::memcpy(T.m, T_h + 12 * h, sizeof(T.m));
    uint32_t c = 0;
    for (size_t i = 0; i < n; i++)
      if (ransac_residual(T, src + 3 * i, dst + 3 * i) <= thresh) c++;
    counts[h] = c;
  }
}

// The sample index sequence of the hypothesis loop (:83-91): partial Fisher-Yates on a permutation
// that PERSISTS across iterations; seed injected in place of std::random_device (:73).
ORC_API void orc_ransac_samples(size_t n, size_t sample_size, size_t iters, uint32_t seed, uint64_t* out) {
  std::vector<size_t> perm(n);
  for (size_t i = 0; i < n; i++) perm[i] = i;
  std::mt19937 rng(seed);
  for (size_t it = 0; it < iters; it++) {
    size_t prev = n;
    for (size_t i = 0; i < sample_size; i++) {
      std::uniform_int_distribution<size_t> dist(0, prev - 1);
      size_t r = dist(rng);
      out[it * sample_size + i] = perm[r];
      prev--;
      std::swap(perm[r], perm[prev]);
    }
  }
}

// estimateModel(sample_ind) (:72-82) for a list of samples -> H hypothesis transforms.
ORC_API void orc_ransac_fit_samples(const float* dst, const float* src, const uint64_t* samples,
                                    size_t sample_size, size_t H, float* T_h) {
  std::vector<float> d(3 * sample_size), s(3 * sample_size);
  for (size_t h = 0; h < H; h++) {
    for (size_t i = 0; i < sample_size; i++)
      for (int r = 0; r < 3; r++) {
        d[3 * i + r] = dst[3 * samples[h * sample_size + i] + r];
        s[3 * i + r] = src[3 * samples[h * sample_size + i] + r];
      }
    T34 T;
    kabsch<float>(d.data(), s.data(), sample_size, T);
    std::memcpy(T_h + 12 * h, T.m, sizeof(T.m));
  }
}

struct orc_ransac_result {
  float T[12];
  uint64_t iterations;
  uint64_t num_inliers;
  uint64_t best_iteration;  // 0-based hypothesis index that produced the kept model
};

ORC_API void orc_ransac_rigid(const float* dst, const float* src, size_t n, uint32_t seed, size_t sample_size,
                              size_t inlier_count_thresh, size_t max_iter, float thresh, int re_estimate,
                              orc_ransac_result* out, uint64_t* inliers /* n */, float* residuals /* n */) {
  if (n < sample_size) sample_size = n;                    // :67
  if (inlier_count_thresh > n) inlier_count_thresh = n;    // :68
  std::vector<size_t> perm(n);
  for (size_t i = 0; i < n; i++) perm[i] = i;
  std::mt19937 rng(seed);
  T34 best = t34_identity();  // the reference's model_params_ is default-constructed (uninitialised
                              // Eigen::Transform); identity is this oracle's stand-in
  std::vector<float> best_res;
  std::vector<size_t> best_inl;
  std::vector<float> cur_res(n);
  std::vector<size_t> cur_inl;
  size_t it = 0, best_it = 0;
  std::vector<float> d(3 * sample_size), s(3 * sample_size);
  while (it < max_iter) {
    std::vector<size_t> samp(sample_size);
    size_t prev = n;
    for (size_t i = 0; i < sample_size; i++) {
      std::uniform_int_distribution<size_t> dist(0, prev - 1);
      size_t r = dist(rng);
      samp[i] = perm[r];
      prev--;
      std::swap(perm[r], perm[prev]);
    }
    for (size_t i = 0; i < sample_size; i++)
      for (int r = 0; r < 3; r++) {
        d[3 * i + r] = dst[3 * samp[i] + r];
        s[3 * i + r] = src[3 * samp[i] + r];
      }
    T34 cur;
    kabsch<float>(d.data(), s.data(), sample_size, cur);
    cur_res.resize(n);
#pragma omp parallel for
    for (size_t i = 0; i < n; i++) cur_res[i] = ransac_residual(cur, src + 3 * i, dst + 3 * i);
    cur_inl.clear();
    for (size_t i = 0; i < n; i++)
      if (cur_res[i] <= thresh) cur_inl.push_back(i);
    it++;
    if (cur_inl.size() < sample_size) continue;  // :104
    if (cur_inl.size() > best_inl.size()) {      // :107-111
      best = cur;
      best_res = cur_res;
      best_inl = cur_inl;
      best_it = it - 1;
    }
    if (best_inl.size() >= inlier_count_thresh) break;  // :114
  }
  if (re_estimate) {  // :118-128
    std::vector<float> dd(3 * best_inl.size()), ss(3 * best_inl.size());
    for (size_t i = 0; i < best_inl.size(); i++)
      for (int r = 0; r < 3; r++) {
        dd[3 * i + r] = dst[3 * best_inl[i] + r];
        ss[3 * i + r] = src[3 * best_inl[i] + r];
      }
    kabsch<float>(dd.data(), ss.data(), best_inl.size(), best);
    best_res.resize(n);
#pragma omp parallel for
    for (size_t i = 0; i < n; i++) best_res[i] = ransac_residual(best, src + 3 * i, dst + 3 * i);
    best_inl.clear();
    for (size_t i = 0; i < n; i++)
      if (best_res[i] <= thresh) best_inl.push_back(i);
  }
  std::memcpy(out->T, best.m, sizeof(best.m));
  out->iterations = it;
  out->num_inliers = best_inl.size();
  out->best_iteration = best_it;
  if (inliers)
    for (size_t i = 0; i < best_inl.size(); i++) inliers[i] = best_inl[i];
  if (residuals && !best_res.empty()) std::memcpy(residuals, best_res.data(), n * sizeof(float));
}

// ---------------------------------------------------------------------------------------------
// Covariance::operator() serial branch — core/covariance.hpp:31-80 (min sample size 2), and
// PrincipalComponentAnalysis::compute_ — core/principal_component_analysis.hpp:76-84.
// cov / evecs are row-major 3x3; evecs columns are the eigenvectors, eigenvalues DESCENDING.
// ---------------------------------------------------------------------------------------------
ORC_API int orc_mean_cov(const float* pts, size_t n, int accum_double, float* mean3, float* cov9) {
  if (n < 2) {
    for (int i = 0; i < 3; i++) mean3[i] = std::numeric_limits<float>::quiet_NaN();
    for (int i = 0; i < 9; i++) cov9[i] = std::numeric_limits<float>::quiet_NaN();
    return 0;
  }
  if (!accum_double) {
    float ms[3] = {0, 0, 0};
    for (size_t i = 0; i < n; i++)
      for (int r = 0; r < 3; r++) ms[r] += pts[3 * i + r];
    const float inv = 1.0f / (float)n;
    for (int r = 0; r < 3; r++) mean3[r] = inv * ms[r];
    float cs[9] = {0};
    for (size_t i = 0; i < n; i++) {
      float t[3] = {pts[3 * i] - mean3[0], pts[3 * i + 1] - mean3[1], pts[3 * i + 2] - mean3[2]};
      for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) cs[r * 3 + c] += t[r] * t[c];
    }
    const float inv1 = 1.0f / (float)(n - 1);
    for (int i = 0; i < 9; i++) cov9[i] = inv1 * cs[i];
  } else {
    double ms[3] = {0, 0, 0};
    for (size_t i = 0; i < n; i++)
      for (int r = 0; r < 3; r++) ms[r] += pts[3 * i + r];
    double mu[3];
    for (int r = 0; r < 3; r++) {
      mu[r] = ms[r] / (double)n;
      mean3[r] = (float)mu[r];
    }
    double cs[9] = {0};
    for (size_t i = 0; i < n; i++) {
      double t[3] = {pts[3 * i] - mu[0], pts[3 * i + 1] - mu[1], pts[3 * i + 2] - mu[2]};
      for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) cs[r * 3 + c] += t[r] * t[c];
    }
    for (int i = 0; i < 9; i++) cov9[i] = (float)(cs[i] / (double)(n - 1));
  }
  return 1;
}

ORC_API int orc_pca(const float* pts, size_t n, int accum_double, float* mean3, float* cov9, float* evals3,
                    float* evecs9) {
  int ok = orc_mean_cov(pts, n, accum_double, mean3, cov9);
  if (!ok) {
    for (int i = 0; i < 3; i++) evals3[i] = std::numeric_limits<float>::quiet_NaN();
    for (int i = 0; i < 9; i++) evecs9[i] = std::numeric_limits<float>::quiet_NaN();
    return 0;
  }
  orc::M3 C, V;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) C.a[r][c] = cov9[r * 3 + c];
  double w[3];
  orc::sym3_eigen(C, w, V);  // ascending, like SelfAdjointEigenSolver
  orc::M3 E;                 // :78 rowwise().reverse() -> descending
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) E.a[r][c] = V.a[r][2 - c];
  if (orc::m3_det(E) < 0.0)  // :79-82 flip the last column
    for (int r = 0; r < 3; r++) E.a[r][2] = -E.a[r][2];
  for (int c = 0; c < 3; c++) evals3[c] = (float)w[2 - c];  // :83
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) evecs9[r * 3 + c] = (float)E.a[r][c];
  return 1;
}

// ---------------------------------------------------------------------------------------------
// Normal (and curvature) estimation from given neighbourhoods — core/normal_estimation.hpp.
// The neighbourhood of point i is nbr[i*stride .. i*stride+cnt[i]) in the order the search returned
// it (ascending distance: KNNSearchResultAdaptor keeps its slots sorted, kd_tree.hpp:77-99; the
// radius adaptor sorts, kd_tree.hpp:130-133); the tests fill it from the reference's own nanoflann
// (oracle/_ref). Per point (normal_estimation.hpp:298-308 / :319-332 / curvature :379-389):
//   * fewer than 3 neighbours (setMinValidSampleSize(points_.rows()), :27/:38; covariance.hpp:93-97)
//     -> NaN normal and curvature;
//   * mean_sum += p sequentially, mean = (1/size) * mean_sum; cov_sum += (p-mean)(p-mean)^T
//     sequentially, cov = (1/(size-1)) * cov_sum — all fp32 (covariance.hpp:121-135), restated
//     bit-exactly (cov6 = xx,xy,xz,yy,yz,zz);
//   * normal = eigenvectors().col(0) of SelfAdjointEigenSolver(cov) (ascending eigenvalues): Eigen is
//     absent from this image, so the eigenvector comes from a double Jacobi (small_linalg.hpp) —
//     parity UNPINNED for this O(1) step; its sign is an artefact of Eigen's QR iteration unless a
//     view point is set, in which case it is flipped when dot(n, view_point - p) < 0 (:325-329);
//   * curvature = eigenvalues()[0] / eigenvalues().sum() (:389).
ORC_API void orc_normals_from_neighbors(const float* pts, size_t n, const int64_t* nbr, size_t stride,
                                        const uint32_t* cnt, const float* view_point3,
                                        const float* ref_normals, float* normals, float* curvature,
                                        float* cov6) {
  const float nan = std::numeric_limits<float>::quiet_NaN();
  const bool use_vp = view_point3 && std::isfinite(view_point3[0]) && std::isfinite(view_point3[1]) &&
                      std::isfinite(view_point3[2]);  // view_point_.allFinite(), :283
#pragma omp parallel for schedule(static)
  for (size_t i = 0; i < n; i++) {
    const size_t m = cnt[i];
    const int64_t* nb = nbr + i * stride;
    if (m < 3) {
      if (normals) normals[3 * i] = normals[3 * i + 1] = normals[3 * i + 2] = nan;
      if (curvature) curvature[i] = nan;
      if (cov6)
        for (int c = 0; c < 6; c++) cov6[6 * i + c] = nan;
      continue;
    }
    float ms[3] = {0.f, 0.f, 0.f};
    for (size_t j = 0; j < m; j++)
      for (int c = 0; c < 3; c++) ms[c] = ms[c] + pts[3 * nb[j] + c];
    const float inv = 1.0f / (float)m;
    const float mean[3] = {inv * ms[0], inv * ms[1], inv * ms[2]};
    float cs[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (size_t j = 0; j < m; j++) {
      const float dx = pts[3 * nb[j]] - mean[0], dy = pts[3 * nb[j] + 1] - mean[1], dz = pts[3 * nb[j] + 2] - mean[2];
      cs[0] = cs[0] + dx * dx;
      cs[1] = cs[1] + dx * dy;
      cs[2] = cs[2] + dx * dz;
      cs[3] = cs[3] + dy * dy;
      cs[4] = cs[4] + dy * dz;
      cs[5] = cs[5] + dz * dz;
    }
    const float invm1 = 1.0f / (float)(m - 1);
    float cv[6];
    for (int c = 0; c < 6; c++) cv[c] = invm1 * cs[c];
    if (cov6)
      for (int c = 0; c < 6; c++) cov6[6 * i + c] = cv[c];
    orc::M3 C, V;
    C.a[0][0] = cv[0]; C.a[0][1] = C.a[1][0] = cv[1]; C.a[0][2] = C.a[2][0] = cv[2];
    C.a[1][1] = cv[3]; C.a[1][2] = C.a[2][1] = cv[4]; C.a[2][2] = cv[5];
    double w[3];
    orc::sym3_eigen(C, w, V);
    float nv[3] = {(float)V.a[0][0], (float)V.a[1][0], (float)V.a[2][0]};
    if (ref_normals) {  // reference normals take precedence (:281-291); flip rule :351-355
      const float* r = ref_normals + 3 * i;
      const float d = nv[0] * r[0] + (nv[1] * r[1] + nv[2] * r[2]);
      if (d < 0.f)
        for (int c = 0; c < 3; c++) nv[c] = -nv[c];
    } else if (use_vp) {
      const float ex = view_point3[0] - pts[3 * i], ey = view_point3[1] - pts[3 * i + 1],
                  ez = view_point3[2] - pts[3 * i + 2];
      const float d = nv[0] * ex + (nv[1] * ey + nv[2] * ez);
      if (d < 0.f)
        for (int c = 0; c < 3; c++) nv[c] = -nv[c];
    }
    if (normals)
      for (int c = 0; c < 3; c++) normals[3 * i + c] = nv[c];
    if (curvature) curvature[i] = (float)(w[0] / (w[0] + w[1] + w[2]));
  }
}

// Brute-force neighbourhoods (stand-in when oracle/_ref is not built): k nearest with d2 < max_d2, or —
// k == 0 — every point with d2 < max_d2, ascending (d2, index); rows truncated to `stride`, cnt = full
// count. Distance arithmetic as nanoflann's L2_Adaptor::evalMetric for dim 3: ((dx^2)+dy^2)+dz^2.
ORC_API void orc_neighborhoods_brute(const float* ref, size_t nr, const float* qry, size_t nq, size_t k,
                                     float max_d2, size_t stride, int64_t* idx, float* d2, uint32_t* cnt) {
#pragma omp parallel for schedule(dynamic, 64)
  for (size_t i = 0; i < nq; i++) {
    std::vector<std::pair<float, int64_t>> c;
    const float qx = qry[3 * i], qy = qry[3 * i + 1], qz = qry[3 * i + 2];
    for (size_t j = 0; j < nr; j++) {
      const float dx = qx - ref[3 * j], dy = qy - ref[3 * j + 1], dz = qz - ref[3 * j + 2];
      const float r = ((dx * dx) + dy * dy) + dz * dz;
      if (r < max_d2) c.emplace_back(r, (int64_t)j);
    }
    std::sort(c.begin(), c.end());
    size_t m = c.size();
    if (k > 0 && m > k) m = k;
    for (size_t j = 0; j < stride; j++) {
      idx[i * stride + j] = j < m ? c[j].second : -1;
      d2[i * stride + j] = j < m ? c[j].first : max_d2;
    }
    cnt[i] = (uint32_t)m;
  }
}

// ---------------------------------------------------------------------------------------------
// Voxel-grid downsampling — PointCloud::gridDownsample (utilities/point_cloud.hpp:246-290) over
// Points[Normals][Colors]GridDownsampler (core/grid_downsampler.hpp) and the SERIAL
// GridAccumulator::build_index_ (core/grid_accumulator.hpp:187-199):
//   * grid coordinate = (ptrdiff_t) std::floor(point[i] * bin_size_inv[i]), bin_size_inv = 1/bin_size
//     in fp32 (:117-126, :87);
//   * std::map keyed by the coordinate triple, lexicographic with x most significant (:9-39);
//   * the first point of a bin builds the accumulator (copy), later points are added in index order:
//     pointSum += p; normalSum +-= n depending on sign(normalSum . n) (common_accumulators.hpp:
//     122-131); colorSum += c;
//   * output per bin with pointCount >= min_points: scale = 1.0f / pointCount, scale * pointSum,
//     (scale * normalSum).normalized(), scale * colorSum (grid_downsampler.hpp:20-37, :97-105).
// order = 0: bins in map order (what the default parallel = true build emits, :177-181 — its SUMS are
// merged across threads in arrival order and are not reproducible; the serial sums are restated);
// order = 1: bins in first-occurrence order (parallel = false, :194-197). Returns the bin count.
ORC_API size_t orc_grid_downsample(const float* pts, const float* nrm, const float* col, size_t n, float bin_size,
                                   size_t min_points, int order, float* out_pts, float* out_nrm, float* out_col) {
  struct Key {
    std::ptrdiff_t c[3];
    bool operator<(const Key& o) const {
      if (c[0] < o.c[0]) return true;
      if (o.c[0] < c[0]) return false;
      if (c[1] < o.c[1]) return true;
      if (o.c[1] < c[1]) return false;
      return c[2] < o.c[2];
    }
  };
  struct Acc {
    float p[3], nv[3], cl[3];
    size_t count;
  };
  const float inv = 1.0f / bin_size;
  std::map<Key, Acc> table;
  std::vector<std::map<Key, Acc>::iterator> seq;
#ifdef _OPENMP
  if (order == 2) {
    // order = 2: the reference's DEFAULT parallel build (grid_accumulator.hpp:149-181) — per-thread
    // private maps over a static partition of the points, merged under a critical section in thread
    // arrival order (mergeWith, common_accumulators.hpp:48-52, :93-103). Same bins and map order as
    // order 0; the sums differ from the serial ones in the last bits and from run to run. Used as the
    // CPU baseline of bench.py and for a tolerance test only.
#pragma omp parallel
    {
      std::map<Key, Acc> priv;
#pragma omp for nowait
      for (size_t i = 0; i < n; i++) {
        Key k;
        for (int a = 0; a < 3; a++) k.c[a] = (std::ptrdiff_t)std::floor(pts[3 * i + a] * inv);
        auto lb = priv.lower_bound(k);
        if (lb != priv.end() && !(k < lb->first)) {
          Acc& acc = lb->second;
          for (int a = 0; a < 3; a++) acc.p[a] = acc.p[a] + pts[3 * i + a];
          if (nrm) {
            const float* v = nrm + 3 * i;
            const float d = sum3(acc.nv[0] * v[0], acc.nv[1] * v[1], acc.nv[2] * v[2]);
            for (int a = 0; a < 3; a++) acc.nv[a] = d < 0.f ? acc.nv[a] - v[a] : acc.nv[a] + v[a];
          }
          if (col)
            for (int a = 0; a < 3; a++) acc.cl[a] = acc.cl[a] + col[3 * i + a];
          acc.count++;
        } else {
          Acc acc;
          for (int a = 0; a < 3; a++) {
            acc.p[a] = pts[3 * i + a];
            acc.nv[a] = nrm ? nrm[3 * i + a] : 0.f;
            acc.cl[a] = col ? col[3 * i + a] : 0.f;
          }
          acc.count = 1;
          priv.emplace_hint(lb, k, acc);
        }
      }
#pragma omp critical
      {
        for (auto it = priv.begin(); it != priv.end(); ++it) {
          auto lb = table.lower_bound(it->first);
          if (lb != table.end() && !(it->first < lb->first)) {
            Acc& acc = lb->second;
            const Acc& o = it->second;
            for (int a = 0; a < 3; a++) acc.p[a] = acc.p[a] + o.p[a];
            const float d = sum3(acc.nv[0] * o.nv[0], acc.nv[1] * o.nv[1], acc.nv[2] * o.nv[2]);
            for (int a = 0; a < 3; a++) acc.nv[a] = d < 0.f ? acc.nv[a] - o.nv[a] : acc.nv[a] + o.nv[a];
            for (int a = 0; a < 3; a++) acc.cl[a] = acc.cl[a] + o.cl[a];
            acc.count += o.count;
          } else {
            table.emplace_hint(lb, it->first, it->second);
          }
        }
      }
    }
    order = 0;
    n = 0;  // skip the serial build below
  }
#endif
  for (size_t i = 0; i < n; i++) {
    Key k;
    for (int a = 0; a < 3; a++) k.c[a] = (std::ptrdiff_t)std::floor(pts[3 * i + a] * inv);
    auto it = table.find(k);
    if (it == table.end()) {
      Acc acc;
      for (int a = 0; a < 3; a++) {
        acc.p[a] = pts[3 * i + a];
        acc.nv[a] = nrm ? nrm[3 * i + a] : 0.f;
        acc.cl[a] = col ? col[3 * i + a] : 0.f;
      }
      acc.count = 1;
      seq.push_back(table.emplace(k, acc).first);
    } else {
      Acc& acc = it->second;
      for (int a = 0; a < 3; a++) acc.p[a] = acc.p[a] + pts[3 * i + a];
      if (nrm) {
        const float* v = nrm + 3 * i;
        const float d = sum3(acc.nv[0] * v[0], acc.nv[1] * v[1], acc.nv[2] * v[2]);
        if (d < 0.f)
          for (int a = 0; a < 3; a++) acc.nv[a] = acc.nv[a] - v[a];
        else
          for (int a = 0; a < 3; a++) acc.nv[a] = acc.nv[a] + v[a];
      }
      if (col)
        for (int a = 0; a < 3; a++) acc.cl[a] = acc.cl[a] + col[3 * i + a];
      acc.count++;
    }
  }
  std::vector<const Acc*> bins;
  if (order == 0)
    for (auto it = table.begin(); it != table.end(); ++it) bins.push_back(&it->second);
  else
    for (auto& it : seq) bins.push_back(&it->second);
  size_t m = 0;
  for (const Acc* b : bins) {
    if (b->count < min_points) continue;
    const float scale = 1.0f / (float)b->count;
    for (int a = 0; a < 3; a++) out_pts[3 * m + a] = scale * b->p[a];
    if (nrm && out_nrm) {
      const float w[3] = {scale * b->nv[0], scale * b->nv[1], scale * b->nv[2]};
      const float z = sum3(w[0] * w[0], w[1] * w[1], w[2] * w[2]);
      if (z > 0.f) {
        const float nn = std::sqrt(z);
        for (int a = 0; a < 3; a++) out_nrm[3 * m + a] = w[a] / nn;
      } else {
        for (int a = 0; a < 3; a++) out_nrm[3 * m + a] = w[a];
      }
    }
    if (col && out_col)
      for (int a = 0; a < 3; a++) out_col[3 * m + a] = scale * b->cl[a];
    m++;
  }
  return m;
}

ORC_API int orc_num_threads() {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

ORC_API void orc_set_num_threads(int n) {
#ifdef _OPENMP
  omp_set_num_threads(n);
#else
  (void)n;
#endif
}
