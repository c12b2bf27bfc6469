// ORACLE — test infrastructure, NOT product code.
//
// Feature-space rigid ICP restated on the CPU: CombinedMetricRigidTransformICP3f<CorrespondenceSearchKDTree<F>> /
// PointToPointMetricRigidTransformICP3f<...> with F = PointNormal / PointColor / PointNormalColorFeaturesAdaptor3f
// (correspondence_search/common_transformable_feature_adaptors.hpp:148-290). Everything except the correspondence
// search is the main restatement's (cilantro_oracle.cpp, compiled into this library as one translation unit so that its
// estimators, filters and loop helpers are used as they are, not copied). Restated here, independently of
// cilantro_b200/csrc/feature_rule.hpp:
//   * the feature vector [p, w_n n, w_c c] (:175-183, :248-259: one fp32 multiply per tail component);
//   * transformFeatures(tform), Isometry branch (:193-204, :269-280): p -> R p + t, w_n n -> R (w_n n), colour copied,
//     with the main oracle's apply() / rotate() (sum3 per row);
//   * the L2 metric, in nanoflann's own loop structure (L2_Adaptor::evalMetric, nanoflann.hpp:570-604): groups of four
//     while four components remain, then one at a time;
//   * the 1-NN by brute force: strict d2 < best over ascending index (lowest index wins exact ties).
// Must be compiled with -ffp-contract=off (the arithmetic contract of cilantro_oracle.cpp).
#include "cilantro_oracle.cpp"

namespace {

inline int feat_tails(int kind) { return kind == 3 ? 2 : (kind == 0 ? 0 : 1); }
inline bool tail_is_normal(int kind, int t) { return t == 0 && (kind == 1 || kind == 3); }

// nanoflann.hpp:570-604 (the early return never changes a strict accept / reject decision)
inline float l2_feature(const float* a, const float* b, size_t D) {
  float result = 0.f;
  size_t d = 0;
  while (d + 3 < D) {
    const float d0 = a[d] - b[d], d1 = a[d + 1] - b[d + 1], d2 = a[d + 2] - b[d + 2], d3 = a[d + 3] - b[d + 3];
    result += d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3;
    d += 4;
  }
  while (d < D) {
    const float d0 = a[d] - b[d];
    result += d0 * d0;
    d++;
  }
  return result;
}

// packed features [p, tails] of n points: D = 3 + 3 * tails floats each
std::vector<float> pack(const float* xyz, const float* tails, size_t n, int nt) {
  const size_t D = 3 + 3 * (size_t)nt;
  std::vector<float> f(D * n);
  for (size_t i = 0; i < n; i++) {
    for (int k = 0; k < 3; k++) f[D * i + k] = xyz[3 * i + k];
    for (int k = 0; k < 3 * nt; k++) f[D * i + 3 + k] = tails[3 * (size_t)nt * i + k];
  }
  return f;
}

// transformFeatures(tform) of packed features
std::vector<float> transform_features(const T34& T, const float* xyz, const float* tails, size_t n, int kind) {
  const int nt = feat_tails(kind);
  const size_t D = 3 + 3 * (size_t)nt;
  std::vector<float> f = pack(xyz, tails, n, nt);
  for (size_t i = 0; i < n; i++) {
    float* x = &f[D * i];
    float q[3];
    apply(T, x, q);
    for (int k = 0; k < 3; k++) x[k] = q[k];
    for (int t = 0; t < nt; t++)
      if (tail_is_normal(kind, t)) {
        rotate(T, x + 3 + 3 * t, q);
        for (int k = 0; k < 3; k++) x[3 + 3 * t + k] = q[k];
      }
  }
  return f;
}

void knn1_feature(const float* ref, size_t nref, const float* qry, size_t nq, size_t D, float max_d2, int64_t* idx,
                  float* d2) {
#pragma omp parallel for schedule(dynamic, 64)
  for (size_t i = 0; i < nq; i++) {
    float best = max_d2;
    int64_t bi = -1;
    for (size_t j = 0; j < nref; j++) {
      const float r = l2_feature(qry + D * i, ref + D * j, D);
      if (r < best) {
        best = r;
        bi = (int64_t)j;
      }
    }
    idx[i] = bi;
    d2[i] = best;
  }
}

// The two searches of one findCorrespondences(T). engine_correspondences() (cilantro_oracle.cpp) calls them through
// its kNN callback (SECOND_TO_FIRST) and its f2s_fn (FIRST_TO_SECOND), which only carry xyz; the feature vectors of the
// current call are reached through g_search. The oracle is driven from one thread (the tests), so one slot suffices.
struct FeatureSearch {
  std::vector<float> dst;      // destination features
  std::vector<float> src_t;    // transformed source features
  size_t D;
};
FeatureSearch* g_search = nullptr;

void s2f_cb(void*, const float*, size_t nq, float max_d2, int64_t* idx, float* d2) {
  knn1_feature(g_search->dst.data(), g_search->dst.size() / g_search->D, g_search->src_t.data(), nq, g_search->D, max_d2,
               idx, d2);
}

void f2s_cb(const float*, size_t nref, const float*, size_t nq, float max_d2, int64_t* idx, float* d2) {
  knn1_feature(g_search->src_t.data(), nref, g_search->dst.data(), nq, g_search->D, max_d2, idx, d2);
}

void feature_correspondences(int kind, const float* dst_p, const float* dst_tails, size_t n_dst, const float* src_p,
                             const float* src_tails, size_t n_src, const T34& T, const orc_icp_params* prm,
                             const float* src_trans, std::vector<Corr>& corr) {
  FeatureSearch fs;
  fs.D = 3 + 3 * (size_t)feat_tails(kind);
  fs.dst = pack(dst_p, dst_tails, n_dst, feat_tails(kind));
  fs.src_t = transform_features(T, src_p, src_tails, n_src, kind);
  g_search = &fs;
  orc_icp_params p = *prm;
  p.f2s_fn = f2s_cb;
  std::vector<int64_t> idx;
  std::vector<float> d2;
  // every configuration goes through the list path, as in the product
  engine_correspondences(dst_p, n_dst, src_trans, n_src, &p, s2f_cb, nullptr, corr, idx, d2);
  g_search = nullptr;
}

}  // namespace

// tails of n points: per point tail 0 = w_n n (normal kinds) then w_c c (colour kinds); out has 3 * tails floats each
ORC_API void orc_feature_tails(int kind, const float* normals, const float* colors, size_t n, float w_n, float w_c,
                               float* out) {
  const int nt = feat_tails(kind);
  for (size_t i = 0; i < n; i++)
    for (int t = 0; t < nt; t++) {
      const bool nrm = tail_is_normal(kind, t);
      const float* v = nrm ? normals + 3 * i : colors + 3 * i;
      const float w = nrm ? w_n : w_c;
      for (int k = 0; k < 3; k++) out[3 * (size_t)nt * i + 3 * t + k] = w * v[k];
    }
}

// 1-NN of packed D-dimensional features (brute force, d2 < max_d2, lowest index on ties)
ORC_API void orc_feature_knn1(const float* ref, size_t nref, const float* qry, size_t nq, size_t D, float max_d2,
                              int64_t* idx, float* d2) {
  knn1_feature(ref, nref, qry, nq, D, max_d2, idx, d2);
}

// transformFeatures(T) of n points: packed D-dimensional features out
ORC_API void orc_transform_features(int kind, const float* T12, const float* xyz, const float* tails, size_t n,
                                    float* out) {
  T34 T;
  std::memcpy(T.m, T12, sizeof(T.m));
  const std::vector<float> f = transform_features(T, xyz, tails, n, kind);
  std::memcpy(out, f.data(), f.size() * sizeof(float));
}

// getCorrespondences() after findCorrespondences(T) with feature adaptors of `kind` and the engine options of prm
ORC_API size_t orc_feature_engine_correspondences(int kind, const float* dst_p, const float* dst_tails, size_t n_dst,
                                                  const float* src_p, const float* src_tails, size_t n_src,
                                                  const float* T12, const orc_icp_params* prm, uint64_t* idx_first,
                                                  uint64_t* idx_second, float* value) {
  T34 T;
  std::memcpy(T.m, T12, sizeof(T.m));
  std::vector<float> q(3 * n_src);
  orc_transform_points(T12, src_p, n_src, q.data());
  std::vector<Corr> corr;
  feature_correspondences(kind, dst_p, dst_tails, n_dst, src_p, src_tails, n_src, T, prm, q.data(), corr);
  for (size_t i = 0; i < corr.size(); i++) {
    idx_first[i] = corr[i].indexInFirst;
    idx_second[i] = corr[i].indexInSecond;
    value[i] = corr[i].value;
  }
  return corr.size();
}

// orc_icp (cilantro_oracle.cpp) with the feature search: same loop, estimators, reorthonormalisation and composition;
// the correspondence values (feature d2) feed the weight evaluators.
ORC_API void orc_feature_icp(int kind, const float* dst_p, const float* dst_n, const float* dst_tails, size_t n_dst,
                             const float* src_p, const float* src_n, const float* src_tails, size_t n_src,
                             const orc_icp_params* prm, orc_icp_result* res, float* T_log) {
  T34 T;
  std::memcpy(T.m, prm->T_init, sizeof(T.m));
  float dst_mean[3] = {0, 0, 0}, src_mean[3] = {0, 0, 0};
  if (prm->metric == 1) {
    colmean(dst_p, n_dst, dst_mean);
    colmean(src_p, n_src, src_mean);
  }
  std::vector<float> src_trans(3 * n_src), src_n_trans;
  if (src_n) src_n_trans.resize(3 * n_src);
  std::vector<Corr> corr;
  int iters = 0;
  float last_delta = std::numeric_limits<float>::infinity();
  while (iters < prm->max_iter) {
    orc_transform_points(T.m, src_p, n_src, src_trans.data());
    feature_correspondences(kind, dst_p, dst_tails, n_dst, src_p, src_tails, n_src, T, prm, src_trans.data(), corr);
    T34 Titer;
    if (prm->metric == 0) {
      if (prm->accum_double)
        kabsch_corr<double>(dst_p, src_trans.data(), corr, Titer);
      else
        kabsch_corr<float>(dst_p, src_trans.data(), corr, Titer);
    } else {
      float src_mean_t[3];
      apply(T, src_mean, src_mean_t);
      const float* sn = nullptr;
      if (src_n) {
        orc_rotate_vectors(T.m, src_n, n_src, src_n_trans.data());
        sn = src_n_trans.data();
      }
      CorrWeights cw;
      cw.pt_kind = prm->pt_weight_kind;
      cw.pl_kind = prm->pl_weight_kind;
      cw.pt_coeff = prm->pt_weight_coeff;
      cw.pl_coeff = prm->pl_weight_coeff;
      if (prm->accum_double)
        estimate_combined<double>(dst_p, dst_n, n_dst, n_dst, src_trans.data(), sn, corr, prm->w_pt, prm->w_pl,
                                  (size_t)prm->max_opt_iter, prm->opt_tol, dst_mean, src_mean_t, prm->parallel != 0,
                                  Titer, cw);
      else
        estimate_combined<float>(dst_p, dst_n, n_dst, n_dst, src_trans.data(), sn, corr, prm->w_pt, prm->w_pl,
                                 (size_t)prm->max_opt_iter, prm->opt_tol, dst_mean, src_mean_t, prm->parallel != 0,
                                 Titer, cw);
    }
    reorthonormalize(Titer);
    T = compose(Titer, T);
    float dn = 0.f;
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) {
        float e = Titer.R(r, c) - (r == c ? 1.f : 0.f);
        dn += e * e;
      }
      dn += Titer.t(r) * Titer.t(r);
    }
    last_delta = std::sqrt(dn);
    if (T_log) std::memcpy(T_log + 12 * iters, T.m, sizeof(T.m));
    iters++;
    if (last_delta < prm->tol) break;
  }
  std::memcpy(res->T, T.m, sizeof(T.m));
  res->iterations = iters;
  res->last_delta = last_delta;
  res->converged = last_delta < prm->tol;
  res->last_num_corr = corr.size();
  res->t_knn_s = 0;
  res->t_est_s = 0;
}
