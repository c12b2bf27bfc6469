// ORACLE (test infrastructure, NOT product code) — the reference's nanoflann on feature vectors.
//
// The kd-tree CorrespondenceSearchKDTree<SearchFeatureAdaptorT> builds over PointNormal / PointColor /
// PointNormalColorFeaturesAdaptor3f features (D = 6 / 9; D = 3 for PointFeaturesAdaptor3f), compiled in place from the
// reference's OWN vendored nanoflann header (never copied into this repo), with the leaf size, build threads and
// result adaptor of nanoflann_ref.cpp (that file is compiled into this library too). Output:
// oracle/_ref/libcilantro_ref_feature_knn.so, built by oracle/Makefile where the reference exists.
#include "nanoflann_ref.cpp"

namespace {

template <int D>
struct PackedFeat {
  std::vector<float> f;
  size_t n;
  inline size_t kdtree_get_point_count() const { return n; }
  inline float kdtree_get_pt(size_t idx, size_t dim) const { return f[D * idx + dim]; }
  template <class BBOX>
  bool kdtree_get_bbox(BBOX&) const { return false; }
};

template <int D>
void knn1(const float* ref, size_t nref, const float* qry, size_t nq, float max_d2, int64_t* idx, float* d2) {
  using Data = PackedFeat<D>;
  using Tree = nanoflann::KDTreeSingleIndexAdaptor<nanoflann::L2_Adaptor<float, Data, float, size_t>, Data, D, size_t>;
  Data data;
  data.f.assign(ref, ref + D * nref);
  data.n = nref;
  if (nref == 0) {
    for (size_t i = 0; i < nq; i++) {
      idx[i] = -1;
      d2[i] = max_d2;
    }
    return;
  }
  Tree tree(D, data, nanoflann::KDTreeSingleIndexAdaptorParams(10, nanoflann::KDTreeSingleIndexAdaptorFlags::None, 1));
  const nanoflann::SearchParameters sp(0.0f, true);
#pragma omp parallel for schedule(dynamic, 256)
  for (size_t i = 0; i < nq; i++) {
    float v;
    size_t ix;
    BoundedKBest rs(&v, &ix, 1, max_d2);
    tree.findNeighbors(rs, qry + D * i, sp);
    idx[i] = rs.size() == 1 ? (int64_t)ix : -1;
    d2[i] = rs.size() == 1 ? v : max_d2;
  }
}

template <int D>
float eval(const float* a, const float* b) {
  PackedFeat<D> data;
  data.f.assign(b, b + D);
  data.n = 1;
  return nanoflann::L2_Adaptor<float, PackedFeat<D>, float, size_t>(data).evalMetric(a, 0, D);
}

}  // namespace

// Radius-bounded 1-NN of packed D-dimensional features (D = 3, 6 or 9) through a kd-tree built over `ref`.
REF_API int ref_feature_knn1(size_t D, const float* ref, size_t nref, const float* qry, size_t nq, float max_d2,
                             int64_t* idx, float* d2) {
  if (D == 3) knn1<3>(ref, nref, qry, nq, max_d2, idx, d2);
  else if (D == 6) knn1<6>(ref, nref, qry, nq, max_d2, idx, d2);
  else if (D == 9) knn1<9>(ref, nref, qry, nq, max_d2, idx, d2);
  else return -1;
  return 0;
}

// L2_Adaptor::evalMetric(a, b) for n pairs of packed D-dimensional vectors (no early return: worst_dist = -1).
REF_API int ref_l2_eval(size_t D, const float* a, const float* b, size_t n, float* out) {
  for (size_t i = 0; i < n; i++) {
    if (D == 3) out[i] = eval<3>(a + 3 * i, b + 3 * i);
    else if (D == 6) out[i] = eval<6>(a + 6 * i, b + 6 * i);
    else if (D == 9) out[i] = eval<9>(a + 9 * i, b + 9 * i);
    else return -1;
  }
  return 0;
}
