// cilantro_b200 — header-only C++ mirror of the cilantro types on the rigid-ICP / k-means / RANSAC /
// PCA hot path, forwarding to the C ABI of libcilantro_b200.so (include/cilantro_b200.h).
//
// Same names, argument meaning and error behaviour as the reference (paths relative to its
// include/cilantro/):
//   VectorSet3f / ConstVectorSetMatrixMap3f / Vector3f      core/data_containers.hpp:73-156
//   RigidTransform3f                                        core/space_transformations.hpp:54-57
//   Neighbor / NeighborSet                                  core/nearest_neighbors.hpp
//   Correspondence / CorrespondenceSet                      core/correspondence.hpp:9-55
//   KDTree3f<>                                              core/kd_tree.hpp:144-397
//   SimplePointToPointMetricRigidICP3f                      registration/icp_common_instances.hpp:250
//   SimpleCombinedMetricRigidICP3f                          registration/icp_common_instances.hpp:261
//   SimpleCombinedMetricDenseRigidWarpFieldICP3f            registration/icp_common_instances.hpp:99-144,284-285
//   TransformSet<RigidTransform3f>, transformPoints         core/space_transformations.hpp:60-136,195-223
//   SimpleCombinedMetricSparseRigidWarpFieldICP3f           registration/icp_common_instances.hpp:146-199,313-314
//   VectorSet<float,3>, KDTree<float,3>, NeighborhoodSet    core/data_containers.hpp, kd_tree.hpp, nearest_neighbors.hpp
//   KMeans3f<>                                              clustering/kmeans.hpp:9-59,205-207
//   RigidTransformRANSACEstimator3f<>                       model_estimation/ransac_transform_estimator.hpp:9-122
//   PrincipalComponentAnalysis3f                            core/principal_component_analysis.hpp:8-89
//   NormalEstimation3f                                      core/normal_estimation.hpp:11-421
//   Points[Normals][Colors]GridDownsampler3f                core/grid_downsampler.hpp:8-340
//   PointCloud3f (points / normals / colors, size, hasNormals, transform, gridDownsample[d], index subsets, remove,
//                 estimateNormals{KNN,Radius,KNNInRadius})  utilities/point_cloud.hpp:14-81,154-199,246-420,557
//   Timer                                                   utilities/timer.hpp
// Eigen3 is an external dependency of cilantro that is absent from the build image, so the containers
// below are minimal Eigen-free stand-ins with the memory layout cilantro uses (column-major 3 x N,
// packed xyz). A cilantro maintainer keeps Eigen and only swaps the method bodies (INTEGRATION.md).
//
// Arbitrary user functors (weight / distance evaluators) cannot cross a C ABI: this path implements
// cilantro's defaults (DistanceEvaluator = identity, UnityWeightEvaluator); anything else is a
// compile-time error here, never a silent CPU fallback.
#pragma once
#include <algorithm>
#include <array>
#include <chrono>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <limits>
#include <memory>
#include <random>
#include <set>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../cilantro_b200.h"
#include "b200_ply.hpp"

// Eigen interoperability (SURVEY 7 step 2): where Eigen is installed, the stand-in containers below convert
// from / to the Eigen types real cilantro code holds (VectorSet<float,3> = Eigen::Matrix<float,3,Dynamic>,
// RigidTransform<float,3> = Eigen::Transform<float,3,Isometry>; core/data_containers.hpp:73-112,155-156,
// core/space_transformations.hpp:54-55). Eigen3 is absent from the image this repo is built and tested in, so this
// block is compiled only on a machine that has it (CILANTRO_B200_NO_EIGEN switches it off explicitly).
#if !defined(CILANTRO_B200_NO_EIGEN) && defined(__has_include)
#if __has_include(<Eigen/Dense>)
#include <Eigen/Dense>
#define CILANTRO_B200_HAS_EIGEN 1
#endif
#endif

namespace cilantro {

// ---- containers -----------------------------------------------------------------------------------
struct Vector3f {
  float v[3] = {0.f, 0.f, 0.f};
  Vector3f() = default;
  Vector3f(float x, float y, float z) : v{x, y, z} {}
  float& operator[](size_t i) { return v[i]; }
  float operator[](size_t i) const { return v[i]; }
  float* data() { return v; }
  const float* data() const { return v; }
  float norm() const { return std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }
};

// Owning 3 x N column-major float matrix (cilantro::VectorSet<float,3>).
class VectorSet3f {
public:
  VectorSet3f() = default;
  VectorSet3f(size_t rows, size_t cols) : d_(3 * cols) { (void)rows; }
  size_t rows() const { return 3; }
  size_t cols() const { return d_.size() / 3; }
  void resize(size_t /*rows*/, size_t cols) { d_.resize(3 * cols); }
  float* data() { return d_.data(); }
  const float* data() const { return d_.data(); }
  float& operator()(size_t r, size_t c) { return d_[3 * c + r]; }
  float operator()(size_t r, size_t c) const { return d_[3 * c + r]; }
  Vector3f col(size_t c) const { return Vector3f(d_[3 * c], d_[3 * c + 1], d_[3 * c + 2]); }
  void setCol(size_t c, const Vector3f& p) {
    d_[3 * c] = p[0];
    d_[3 * c + 1] = p[1];
    d_[3 * c + 2] = p[2];
  }
#ifdef CILANTRO_B200_HAS_EIGEN
  // same memory layout as Eigen::Matrix<float, 3, Dynamic> (column-major, packed xyz)
  VectorSet3f(const Eigen::Matrix<float, 3, Eigen::Dynamic>& m) : d_(m.data(), m.data() + 3 * m.cols()) {}
  Eigen::Map<Eigen::Matrix<float, 3, Eigen::Dynamic>> eigen() { return {d_.data(), 3, (Eigen::Index)cols()}; }
  Eigen::Map<const Eigen::Matrix<float, 3, Eigen::Dynamic>> eigen() const { return {d_.data(), 3, (Eigen::Index)cols()}; }
  operator Eigen::Matrix<float, 3, Eigen::Dynamic>() const { return eigen(); }
#endif

private:
  std::vector<float> d_;
};

// Non-owning view (cilantro::ConstVectorSetMatrixMap<float,3>): implicit from the same sources as
// the reference's (VectorSet, std::vector<float>, std::vector<Vector3f>, raw pointer + count).
class ConstVectorSetMatrixMap3f {
public:
  ConstVectorSetMatrixMap3f(const float* data = nullptr, size_t n = 0) : p_(data), n_(n) {}
  ConstVectorSetMatrixMap3f(const VectorSet3f& s) : p_(s.data()), n_(s.cols()) {}
  ConstVectorSetMatrixMap3f(const std::vector<float>& s) : p_(s.data()), n_(s.size() / 3) {}
  ConstVectorSetMatrixMap3f(const std::vector<Vector3f>& s)
      : p_(s.empty() ? nullptr : s[0].data()), n_(s.size()) {}
#ifdef CILANTRO_B200_HAS_EIGEN
  // the sources ConstVectorSetMatrixMap<float,3> accepts in the reference (core/data_containers.hpp:73-112)
  ConstVectorSetMatrixMap3f(const Eigen::Matrix<float, 3, Eigen::Dynamic>& m) : p_(m.data()), n_((size_t)m.cols()) {}
  ConstVectorSetMatrixMap3f(const Eigen::Map<const Eigen::Matrix<float, 3, Eigen::Dynamic>>& m)
      : p_(m.data()), n_((size_t)m.cols()) {}
  ConstVectorSetMatrixMap3f(const Eigen::Map<Eigen::Matrix<float, 3, Eigen::Dynamic>>& m)
      : p_(m.data()), n_((size_t)m.cols()) {}
  ConstVectorSetMatrixMap3f(const std::vector<Eigen::Vector3f>& s)
      : p_(s.empty() ? nullptr : s[0].data()), n_(s.size()) {}
  Eigen::Map<const Eigen::Matrix<float, 3, Eigen::Dynamic>> eigen() const { return {p_, 3, (Eigen::Index)n_}; }
#endif
  const float* data() const { return p_; }
  size_t cols() const { return n_; }
  size_t rows() const { return 3; }
  Vector3f col(size_t c) const { return Vector3f(p_[3 * c], p_[3 * c + 1], p_[3 * c + 2]); }

private:
  const float* p_;
  size_t n_;
};

// Rigid transform, row-major [R | t] storage; the accessor surface of Eigen::Transform<float,3,Isometry>
// that cilantro's examples use.
class RigidTransform3f {
public:
  RigidTransform3f() { setIdentity(); }
  explicit RigidTransform3f(const float* T12) { std::memcpy(m_, T12, sizeof(m_)); }
  static RigidTransform3f Identity() { return RigidTransform3f(); }
  void setIdentity() {
    for (float& x : m_) x = 0.f;
    m_[0] = m_[5] = m_[10] = 1.f;
  }
  float& linear(size_t r, size_t c) { return m_[4 * r + c]; }
  float linear(size_t r, size_t c) const { return m_[4 * r + c]; }
  float& translation(size_t r) { return m_[4 * r + 3]; }
  float translation(size_t r) const { return m_[4 * r + 3]; }
  const float* data() const { return m_; }
  float* data() { return m_; }
  std::array<float, 16> matrix() const {
    std::array<float, 16> M{};
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 4; c++) M[4 * r + c] = m_[4 * r + c];
    M[15] = 1.f;
    return M;
  }
  Vector3f operator*(const Vector3f& p) const {
    Vector3f q;
    for (int r = 0; r < 3; r++) q[r] = (m_[4 * r] * p[0] + (m_[4 * r + 1] * p[1] + m_[4 * r + 2] * p[2])) + m_[4 * r + 3];
    return q;
  }
  RigidTransform3f operator*(const RigidTransform3f& o) const {
    RigidTransform3f r;
    cb_compose(m_, o.m_, r.m_);
    return r;
  }
  RigidTransform3f inverse() const {
    RigidTransform3f r;
    for (int i = 0; i < 3; i++) {
      for (int j = 0; j < 3; j++) r.m_[4 * i + j] = m_[4 * j + i];
      r.m_[4 * i + 3] = -(m_[i] * m_[3] + m_[4 + i] * m_[7] + m_[8 + i] * m_[11]);
    }
    return r;
  }
#ifdef CILANTRO_B200_HAS_EIGEN
  // cilantro::RigidTransform<float,3> = Eigen::Transform<float,3,Eigen::Isometry> (core/space_transformations.hpp:54-55)
  RigidTransform3f(const Eigen::Transform<float, 3, Eigen::Isometry>& T) {
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) m_[4 * r + c] = T.linear()(r, c);
      m_[4 * r + 3] = T.translation()(r);
    }
  }
  operator Eigen::Transform<float, 3, Eigen::Isometry>() const {
    Eigen::Transform<float, 3, Eigen::Isometry> T = Eigen::Transform<float, 3, Eigen::Isometry>::Identity();
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) T.linear()(r, c) = m_[4 * r + c];
      T.translation()(r) = m_[4 * r + 3];
    }
    return T;
  }
#endif

private:
  float m_[12];
};

template <typename ScalarT = float, typename IndexT = size_t>
struct Neighbor {
  IndexT index;
  ScalarT value;
};
template <typename ScalarT = float, typename IndexT = size_t>
using NeighborSet = std::vector<Neighbor<ScalarT, IndexT>>;
template <typename ScalarT = float, typename IndexT = size_t>
using Neighborhood = NeighborSet<ScalarT, IndexT>;
template <typename ScalarT = float, typename IndexT = size_t>
using NeighborhoodSet = std::vector<NeighborSet<ScalarT, IndexT>>;  // core/nearest_neighbors.hpp

// neighbourhood specifications (core/nearest_neighbors.hpp:58-87); radii are squared distances
template <typename CountT = size_t>
struct KNNNeighborhoodSpecification {
  KNNNeighborhoodSpecification(CountT k = (CountT)0) : maxNumberOfNeighbors(k) {}
  CountT maxNumberOfNeighbors;
};
template <typename ScalarT>
struct RadiusNeighborhoodSpecification {
  RadiusNeighborhoodSpecification(ScalarT r = (ScalarT)0) : radius(r) {}
  ScalarT radius;
};
template <typename ScalarT, typename CountT = size_t>
struct KNNInRadiusNeighborhoodSpecification {
  KNNInRadiusNeighborhoodSpecification(CountT k = 0, ScalarT r = (ScalarT)0) : maxNumberOfNeighbors(k), radius(r) {}
  CountT maxNumberOfNeighbors;
  ScalarT radius;
};

template <typename ScalarT = float, typename IndexT = size_t>
struct Correspondence {
  IndexT indexInFirst;
  IndexT indexInSecond;
  ScalarT value;
};
template <typename ScalarT = float, typename IndexT = size_t>
using CorrespondenceSet = std::vector<Correspondence<ScalarT, IndexT>>;

class Timer {  // utilities/timer.hpp:7-43
public:
  void start() { t0_ = std::chrono::high_resolution_clock::now(); }
  void stop() { t1_ = std::chrono::high_resolution_clock::now(); }
  double getElapsedTime() const { return std::chrono::duration<double, std::milli>(t1_ - t0_).count(); }

private:
  std::chrono::high_resolution_clock::time_point t0_, t1_;
};

// ---- library plumbing -------------------------------------------------------------------------------
namespace b200 {

inline void check(int rc, const char* what) {
  if (rc < 0) throw std::runtime_error(std::string(what) + ": " + cb_last_error());
}

// the reference seeds from std::random_device (kmeans.hpp:41, ransac_base.hpp:73); so does the
// default here, and setRandomSeed() / the seed argument make runs reproducible
inline uint32_t random_seed() { return std::random_device{}(); }

// One context per process and device (cb_context is not thread-safe: like the reference's objects,
// use one thread per set of objects).
class Context {
public:
  static cb_context* get(int device = 0) {
    static Context c(device);
    return c.ctx_;
  }

private:
  explicit Context(int device) { check(cb_context_create(device, &ctx_), "cb_context_create"); }
  ~Context() { /* process lifetime; objects holding clouds may outlive static destruction order */ }
  cb_context* ctx_ = nullptr;
};

struct CloudHandle {
  cb_cloud* h = nullptr;
  CloudHandle() = default;
  CloudHandle(const ConstVectorSetMatrixMap3f& pts, const ConstVectorSetMatrixMap3f* normals = nullptr) {
    reset(pts, normals);
  }
  void reset(const ConstVectorSetMatrixMap3f& pts, const ConstVectorSetMatrixMap3f* normals = nullptr) {
    if (h) cb_cloud_destroy(h);
    h = nullptr;
    const float* n = (normals && normals->cols() == pts.cols() && pts.cols() > 0) ? normals->data() : nullptr;
    check(cb_cloud_create(Context::get(), pts.data(), n, pts.cols(), 0, &h), "cb_cloud_create");
  }
  CloudHandle(CloudHandle&& o) noexcept : h(o.h) { o.h = nullptr; }
  CloudHandle(const CloudHandle&) = delete;
  CloudHandle& operator=(const CloudHandle&) = delete;
  ~CloudHandle() {
    if (h) cb_cloud_destroy(h);
  }
};

}  // namespace b200

// ---- KDTree3f<> ------------------------------------------------------------------------------------
// The "tree" is the device-resident uniform grid; queries are exact (same result set as the kd-tree,
// ties broken on the lower index).
template <typename IndexT = size_t>
class KDTree3f {
public:
  using NeighborResult = Neighbor<float, IndexT>;
  using NeighborhoodResult = NeighborSet<float, IndexT>;
  using NeighborhoodSetResult = std::vector<NeighborhoodResult>;

  KDTree3f(const ConstVectorSetMatrixMap3f& data, size_t /*max_leaf_size*/ = 10, size_t /*num_build_threads*/ = 1)
      : n_(data.cols()), data_map_(data), cloud_(data) {}

  bool isEmpty() const { return n_ == 0; }

  // single-point queries (core/kd_tree.hpp:181-193, 215-230, 283-299)
  NeighborResult nearestNeighborSearch(const Vector3f& q) const {
    NeighborhoodResult r = kNNInRadiusSearch(q, 1, std::numeric_limits<float>::max());
    if (r.empty()) throw std::runtime_error("nearestNeighborSearch on an empty tree");  // nanoflann.hpp:1715-1718
    return r[0];
  }
  NeighborhoodResult kNNSearch(const Vector3f& q, size_t k) const {
    return kNNInRadiusSearch(q, k, std::numeric_limits<float>::max());
  }
  NeighborhoodResult kNNInRadiusSearch(const Vector3f& q, size_t k, float radius) const {
    NeighborhoodSetResult r = kNNInRadiusSearch(ConstVectorSetMatrixMap3f(q.data(), 1), k, radius);
    return r.empty() ? NeighborhoodResult() : r[0];
  }
  // batched queries (core/kd_tree.hpp:196-213, 232-249, 301-318)
  NeighborhoodResult nearestNeighborSearch(const ConstVectorSetMatrixMap3f& queries) const {
    std::vector<int64_t> idx(queries.cols());
    std::vector<float> d2(queries.cols());
    b200::CloudHandle q(queries);
    b200::check(cb_knn1_radius(b200::Context::get(), cloud_.h, q.h, nullptr, std::numeric_limits<float>::max(),
                               idx.data(), d2.data()),
                "cb_knn1_radius");
    NeighborhoodResult out(queries.cols());
    for (size_t i = 0; i < out.size(); i++) out[i] = {static_cast<IndexT>(idx[i]), d2[i]};
    return out;
  }
  NeighborhoodSetResult kNNSearch(const ConstVectorSetMatrixMap3f& queries, size_t k) const {
    return kNNInRadiusSearch(queries, k, std::numeric_limits<float>::max());
  }
  NeighborhoodSetResult kNNInRadiusSearch(const ConstVectorSetMatrixMap3f& queries, size_t k, float radius) const {
    const size_t nq = queries.cols();
    NeighborhoodSetResult out(nq);
    if (nq == 0 || k == 0 || n_ == 0) return out;
    if (k > 256) throw std::runtime_error("cilantro_b200: kNN supports k <= 256");
    std::vector<int64_t> idx(nq * k);
    std::vector<float> d2(nq * k);
    std::vector<uint32_t> cnt(nq);
    b200::CloudHandle q(queries);
    b200::check(cb_knn_radius(b200::Context::get(), cloud_.h, q.h, nullptr, (int)k, radius, idx.data(), d2.data(),
                              cnt.data()),
                "cb_knn_radius");
    for (size_t i = 0; i < nq; i++) {
      out[i].resize(cnt[i]);
      for (uint32_t j = 0; j < cnt[i]; j++) out[i][j] = {static_cast<IndexT>(idx[i * k + j]), d2[i * k + j]};
    }
    return out;
  }
  // radiusSearch (core/kd_tree.hpp:250-278): every point with squared distance < radius, ascending distance
  NeighborhoodSetResult radiusSearch(const ConstVectorSetMatrixMap3f& queries, float radius) const {
    const size_t nq = queries.cols();
    NeighborhoodSetResult out(nq);
    if (nq == 0 || n_ == 0) return out;
    b200::CloudHandle q(queries);
    std::vector<uint64_t> off(nq + 1);
    size_t total = 0;
    b200::check(cb_radius_search(b200::Context::get(), cloud_.h, q.h, nullptr, radius, off.data(), nullptr, nullptr, 0,
                                 &total),
                "cb_radius_search");
    if (total == 0) return out;
    std::vector<int64_t> idx(total);
    std::vector<float> d2(total);
    b200::check(cb_radius_search(b200::Context::get(), cloud_.h, q.h, nullptr, radius, off.data(), idx.data(), d2.data(),
                                 total, &total),
                "cb_radius_search");
    for (size_t i = 0; i < nq; i++) {
      out[i].resize(off[i + 1] - off[i]);
      for (size_t j = off[i]; j < off[i + 1]; j++) out[i][j - off[i]] = {static_cast<IndexT>(idx[j]), d2[j]};
    }
    return out;
  }
  NeighborhoodResult radiusSearch(const Vector3f& q, float radius) const {
    NeighborhoodSetResult r = radiusSearch(ConstVectorSetMatrixMap3f(q.data(), 1), radius);
    return r.empty() ? NeighborhoodResult() : r[0];
  }
  // search(query / queries, neighbourhood specification) (core/kd_tree.hpp:320-381)
  template <typename QueryT, typename CountT>
  auto search(const QueryT& q, const KNNNeighborhoodSpecification<CountT>& nh) const {
    return kNNSearch(q, (size_t)nh.maxNumberOfNeighbors);
  }
  template <typename QueryT>
  auto search(const QueryT& q, const RadiusNeighborhoodSpecification<float>& nh) const {
    return radiusSearch(q, nh.radius);
  }
  template <typename QueryT, typename CountT>
  auto search(const QueryT& q, const KNNInRadiusNeighborhoodSpecification<float, CountT>& nh) const {
    return kNNInRadiusSearch(q, (size_t)nh.maxNumberOfNeighbors, nh.radius);
  }
  // the form with an output argument (core/kd_tree.hpp:320-381), as the reference's examples call it
  template <typename SpecT>
  void search(const ConstVectorSetMatrixMap3f& queries, const SpecT& nh, NeighborhoodSetResult& result) const {
    result = search(queries, nh);
  }
  const ConstVectorSetMatrixMap3f& getPointsMatrixMap() const { return data_map_; }  // core/kd_tree.hpp:172-174
  cb_cloud* b200_cloud() const { return cloud_.h; }  // the device-resident cloud (reused by ConnectedComponentExtraction3f)

private:
  size_t n_;
  ConstVectorSetMatrixMap3f data_map_;
  b200::CloudHandle cloud_;
};

// VectorSet<float, 3> and KDTree<float, 3> (core/data_containers.hpp, core/kd_tree.hpp): the 3-D float instances are
// the only ones; any other scalar or dimension is a compile-time error.
namespace b200 {
template <class ScalarT, long EigenDim>
struct Instance3f {
  static_assert(sizeof(ScalarT) == 0, "cilantro_b200 provides the <float, 3> instances only");
};
template <>
struct Instance3f<float, 3> {
  using VectorSet = VectorSet3f;
  using KDTree = KDTree3f<>;
};
}  // namespace b200
template <class ScalarT, long EigenDim>
using VectorSet = typename b200::Instance3f<ScalarT, EigenDim>::VectorSet;
template <class ScalarT, long EigenDim, class... DistanceAdaptorT>
using KDTree = typename b200::Instance3f<ScalarT, EigenDim>::KDTree;

// ---- ICP ---------------------------------------------------------------------------------------------
enum struct CorrespondenceSearchDirection { FIRST_TO_SECOND, SECOND_TO_FIRST, BOTH };

// CorrespondenceSearchKDTree's fluent surface (correspondence_search/correspondence_search_kd_tree.hpp:237-285).
// The defaults run the fused kernel; any other setting goes through the device-side list (icp_engine.cu).
class CorrespondenceSearchEngineB200 {
public:
  using SearchResult = CorrespondenceSet<float, size_t>;
  float getMaxDistance() const { return max_distance_; }
  CorrespondenceSearchEngineB200& setMaxDistance(float dist_thresh_squared) {
    max_distance_ = dist_thresh_squared;
    return *this;
  }
  const CorrespondenceSearchDirection& getSearchDirection() const { return dir_; }
  CorrespondenceSearchEngineB200& setSearchDirection(const CorrespondenceSearchDirection& d) {
    dir_ = d;
    return *this;
  }
  double getInlierFraction() const { return inlier_fraction_; }
  CorrespondenceSearchEngineB200& setInlierFraction(double fraction) {
    inlier_fraction_ = fraction;
    return *this;
  }
  bool getRequireReciprocality() const { return require_reciprocality_; }
  CorrespondenceSearchEngineB200& setRequireReciprocality(bool require_reciprocal) {
    require_reciprocality_ = require_reciprocal;
    return *this;
  }
  bool getOneToOne() const { return one_to_one_; }
  CorrespondenceSearchEngineB200& setOneToOne(bool one_to_one) {
    one_to_one_ = one_to_one;
    return *this;
  }
  const SearchResult& getCorrespondences() const { return corr_; }
  void fill(cb_icp_params& p) const {
    p.max_d2 = max_distance_;
    p.search_dir = dir_ == CorrespondenceSearchDirection::SECOND_TO_FIRST
                       ? CB_SECOND_TO_FIRST
                       : (dir_ == CorrespondenceSearchDirection::FIRST_TO_SECOND ? CB_FIRST_TO_SECOND : CB_BOTH);
    p.inlier_fraction = inlier_fraction_;
    p.require_reciprocal = require_reciprocality_ ? 1 : 0;
    p.one_to_one = one_to_one_ ? 1 : 0;
  }

private:
  template <int>
  friend class SimpleRigidICP3fB200;
  float max_distance_ = (float)(0.01 * 0.01);  // correspondence_search_kd_tree.hpp:49
  CorrespondenceSearchDirection dir_ = CorrespondenceSearchDirection::SECOND_TO_FIRST;
  double inlier_fraction_ = 1.0;
  bool require_reciprocality_ = false;
  bool one_to_one_ = false;
  SearchResult corr_;
};

template <int kMetric>
class SimpleRigidICP3fB200 {
public:
  using Transform = RigidTransform3f;

  // point-to-point: (dst, src); combined: (dst, dst_normals, src[, src_normals])
  SimpleRigidICP3fB200(const ConstVectorSetMatrixMap3f& dst, const ConstVectorSetMatrixMap3f& src) {
    upload(dst, nullptr, src, nullptr);
    init();
  }
  SimpleRigidICP3fB200(const ConstVectorSetMatrixMap3f& dst, const ConstVectorSetMatrixMap3f& dst_n,
                       const ConstVectorSetMatrixMap3f& src) {
    upload(dst, &dst_n, src, nullptr);
    init();
  }
  SimpleRigidICP3fB200(const ConstVectorSetMatrixMap3f& dst, const ConstVectorSetMatrixMap3f& dst_n,
                       const ConstVectorSetMatrixMap3f& src, const ConstVectorSetMatrixMap3f& src_n) {
    upload(dst, &dst_n, src, &src_n);
    init();
  }
  ~SimpleRigidICP3fB200() {
    if (icp_) cb_icp_destroy(icp_);
  }
  SimpleRigidICP3fB200(const SimpleRigidICP3fB200&) = delete;

  CorrespondenceSearchEngineB200& correspondenceSearchEngine() { return engine_; }
  const CorrespondenceSearchEngineB200& correspondenceSearchEngine() const { return engine_; }

  // IterativeClosestPointBase surface (registration/icp_base.hpp:40-106)
  size_t getMaxNumberOfIterations() const { return prm_.max_iter; }
  SimpleRigidICP3fB200& setMaxNumberOfIterations(size_t n) {
    prm_.max_iter = (int32_t)n;
    return *this;
  }
  size_t getNumberOfPerformedIterations() const { return res_.iterations; }
  float getConvergenceTolerance() const { return prm_.tol; }
  SimpleRigidICP3fB200& setConvergenceTolerance(float tol) {
    prm_.tol = tol;
    return *this;
  }
  RigidTransform3f getInitialTransform() const { return RigidTransform3f(prm_.T_init); }
  SimpleRigidICP3fB200& setInitialTransform(const RigidTransform3f& T) {
    std::memcpy(prm_.T_init, T.data(), sizeof(prm_.T_init));
    return *this;
  }
  float getLastUpdateNorm() const { return res_.last_delta; }
  bool hasConverged() const { return res_.last_delta < prm_.tol; }
  const RigidTransform3f& getTransform() const { return T_; }

  // CombinedMetricSingleTransformICP surface (icp_single_transform_combined_metric.hpp:103-141)
  float getPointToPointMetricWeight() const { return prm_.w_pt; }
  SimpleRigidICP3fB200& setPointToPointMetricWeight(float w) {
    prm_.w_pt = w;
    return *this;
  }
  float getPointToPlaneMetricWeight() const { return prm_.w_pl; }
  SimpleRigidICP3fB200& setPointToPlaneMetricWeight(float w) {
    prm_.w_pl = w;
    return *this;
  }
  size_t getMaxNumberOfOptimizationStepIterations() const { return prm_.max_opt_iter; }
  SimpleRigidICP3fB200& setMaxNumberOfOptimizationStepIterations(size_t n) {
    prm_.max_opt_iter = (int32_t)n;
    return *this;
  }
  float getOptimizationStepConvergenceTolerance() const { return prm_.opt_tol; }
  SimpleRigidICP3fB200& setOptimizationStepConvergenceTolerance(float tol) {
    prm_.opt_tol = tol;
    return *this;
  }

  SimpleRigidICP3fB200& estimate() {
    engine_.fill(prm_);
    b200::check(cb_icp_estimate(icp_, &prm_, &res_), "cb_icp_estimate");
    T_ = RigidTransform3f(res_.T);
    corr_fresh_ = false;
    return *this;
  }
  SimpleRigidICP3fB200& estimate(size_t max_iter, float conv_tol) {
    prm_.max_iter = (int32_t)max_iter;
    prm_.tol = conv_tol;
    return estimate();
  }

  // correspondenceSearchEngine().getCorrespondences() after estimate(): materialised on demand
  const CorrespondenceSet<float, size_t>& getCorrespondences() {
    if (!corr_fresh_) {
      const size_t n = cb_cloud_size(src_.h) + cb_cloud_size(dst_.h);
      std::vector<uint64_t> a(n), b(n);
      std::vector<float> v(n);
      size_t cnt = 0;
      b200::check(cb_icp_correspondences(icp_, a.data(), b.data(), v.data(), &cnt), "cb_icp_correspondences");
      engine_.corr_.resize(cnt);
      for (size_t i = 0; i < cnt; i++) engine_.corr_[i] = {(size_t)a[i], (size_t)b[i], v[i]};
      corr_fresh_ = true;
    }
    return engine_.corr_;
  }

  // getResiduals() -> computeResiduals() (icp_base.hpp:102-104): 1 x N_src
  std::vector<float> getResiduals() {
    std::vector<float> r(cb_cloud_size(src_.h));
    prm_.max_d2 = engine_.max_distance_;
    b200::check(cb_icp_residuals(icp_, &prm_, T_.data(), r.data()), "cb_icp_residuals");
    return r;
  }

  double getLastEstimateDeviceMilliseconds() const { return res_.gpu_ms_total; }

protected:
  cb_icp_params& params() { return prm_; }
  cb_icp* b200_icp() { return icp_; }

private:
  // both clouds in one call: the source upload overlaps the destination's grid build (cb_cloud_create_pair)
  void upload(const ConstVectorSetMatrixMap3f& dst, const ConstVectorSetMatrixMap3f* dst_n,
              const ConstVectorSetMatrixMap3f& src, const ConstVectorSetMatrixMap3f* src_n) {
    const float* dn = (dst_n && dst_n->cols() == dst.cols() && dst.cols() > 0) ? dst_n->data() : nullptr;
    const float* sn = (src_n && src_n->cols() == src.cols() && src.cols() > 0) ? src_n->data() : nullptr;
    b200::check(cb_cloud_create_pair(b200::Context::get(), dst.data(), dn, dst.cols(), 0, src.data(), sn, src.cols(), 0,
                                     &dst_.h, &src_.h),
                "cb_cloud_create_pair");
  }
  void init() {
    cb_icp_default_params(&prm_);
    prm_.metric = kMetric;
    std::memset(&res_, 0, sizeof(res_));
    res_.last_delta = std::numeric_limits<float>::infinity();
    b200::check(cb_icp_create(b200::Context::get(), dst_.h, src_.h, &icp_), "cb_icp_create");
  }
  b200::CloudHandle dst_, src_;
  cb_icp* icp_ = nullptr;
  cb_icp_params prm_;
  cb_icp_result res_;
  RigidTransform3f T_;
  CorrespondenceSearchEngineB200 engine_;
  bool corr_fresh_ = false;
};

using SimplePointToPointMetricRigidICP3f = SimpleRigidICP3fB200<CB_ICP_POINT_TO_POINT>;
using SimpleCombinedMetricRigidICP3f = SimpleRigidICP3fB200<CB_ICP_COMBINED>;

// ---- correspondence weight evaluators (core/common_pair_evaluators.hpp) ---------------------------------------
// The two evaluators a C ABI can carry, by kind + coefficient (cb_icp_params::pt_weight_kind ...). Same class names
// and setters as the reference; operator() is kept so that host-side code calling the evaluator still compiles.
template <typename ValueT = float, typename WeightT = ValueT>
class UnityWeightEvaluator {  // :29-43
public:
  using InputScalar = ValueT;
  using OutputScalar = WeightT;
  constexpr WeightT operator()(ValueT) const { return (WeightT)1; }
  template <class PointT>
  constexpr WeightT operator()(const PointT&, const PointT&, ValueT) const { return (WeightT)1; }
  constexpr WeightT operator()(size_t, size_t, ValueT) const { return (WeightT)1; }
  static constexpr int b200_kind() { return CB_WEIGHT_UNITY; }
  float b200_coeff() const { return 0.f; }
};

template <typename ValueT = float, typename WeightT = ValueT, bool distances_are_squared = true>
class RBFKernelWeightEvaluator {  // :46-79
  static_assert(distances_are_squared, "ICP correspondences carry squared distances: only the <.., true> evaluator maps to the device path");

public:
  using InputScalar = ValueT;
  using OutputScalar = WeightT;
  RBFKernelWeightEvaluator() : coeff_(-(WeightT)(0.5)) {}
  RBFKernelWeightEvaluator(ValueT sigma) : coeff_(-(WeightT)(0.5) / (sigma * sigma)) {}
  RBFKernelWeightEvaluator& setSigma(ValueT sigma) {
    coeff_ = -(WeightT)(0.5) / (sigma * sigma);
    return *this;
  }
  WeightT operator()(ValueT dist) const { return std::exp(coeff_ * static_cast<WeightT>(dist)); }
  template <class PointT>
  WeightT operator()(const PointT&, const PointT&, ValueT dist) const { return std::exp(coeff_ * static_cast<WeightT>(dist)); }
  WeightT operator()(size_t, size_t, ValueT dist) const { return std::exp(coeff_ * static_cast<WeightT>(dist)); }
  static constexpr int b200_kind() { return CB_WEIGHT_RBF; }
  float b200_coeff() const { return (float)coeff_; }

private:
  WeightT coeff_;
};

// CombinedMetricRigidICP3f<CorrSearchT, PointToPointCorrWeightEvaluatorT, PointToPlaneCorrWeightEvaluatorT>
// (registration/icp_common_instances.hpp:29-31 over icp_single_transform_combined_metric.hpp:9-101): the general form
// with caller-owned evaluators, held by reference like the reference does (their sigma is read at every estimate()).
// The correspondence search engine argument of the reference is this object's own engine
// (correspondenceSearchEngine()); any evaluator type other than the two above is a compile-time error.
template <class PointToPointCorrWeightEvaluatorT = UnityWeightEvaluator<float, float>,
          class PointToPlaneCorrWeightEvaluatorT = UnityWeightEvaluator<float, float>>
class CombinedMetricRigidICP3f : public SimpleRigidICP3fB200<CB_ICP_COMBINED> {
  using Base = SimpleRigidICP3fB200<CB_ICP_COMBINED>;

public:
  using PointToPointCorrespondenceWeightEvaluator = PointToPointCorrWeightEvaluatorT;
  using PointToPlaneCorrespondenceWeightEvaluator = PointToPlaneCorrWeightEvaluatorT;
  CombinedMetricRigidICP3f(const ConstVectorSetMatrixMap3f& dst, const ConstVectorSetMatrixMap3f& dst_n,
                           const ConstVectorSetMatrixMap3f& src, PointToPointCorrWeightEvaluatorT& point_corr_eval,
                           PointToPlaneCorrWeightEvaluatorT& plane_corr_eval)
      : Base(dst, dst_n, src), pt_(point_corr_eval), pl_(plane_corr_eval) {}
  CombinedMetricRigidICP3f(const ConstVectorSetMatrixMap3f& dst, const ConstVectorSetMatrixMap3f& dst_n,
                           const ConstVectorSetMatrixMap3f& src, const ConstVectorSetMatrixMap3f& src_n,
                           PointToPointCorrWeightEvaluatorT& point_corr_eval, PointToPlaneCorrWeightEvaluatorT& plane_corr_eval)
      : Base(dst, dst_n, src, src_n), pt_(point_corr_eval), pl_(plane_corr_eval) {}
  PointToPointCorrWeightEvaluatorT& pointToPointCorrespondenceWeightEvaluator() { return pt_; }
  PointToPlaneCorrWeightEvaluatorT& pointToPlaneCorrespondenceWeightEvaluator() { return pl_; }
  CombinedMetricRigidICP3f& estimate() {
    this->params().pt_weight_kind = PointToPointCorrWeightEvaluatorT::b200_kind();
    this->params().pl_weight_kind = PointToPlaneCorrWeightEvaluatorT::b200_kind();
    this->params().pt_weight_coeff = pt_.b200_coeff();
    this->params().pl_weight_coeff = pl_.b200_coeff();
    Base::estimate();
    return *this;
  }
  CombinedMetricRigidICP3f& estimate(size_t max_iter, float conv_tol) {
    this->setMaxNumberOfIterations(max_iter);
    this->setConvergenceTolerance(conv_tol);
    return estimate();
  }

private:
  PointToPointCorrWeightEvaluatorT& pt_;
  PointToPlaneCorrWeightEvaluatorT& pl_;
};

// ---- feature-space correspondence search (correspondence_search/common_transformable_feature_adaptors.hpp,
// correspondence_search_kd_tree.hpp, registration/icp_common_instances.hpp:262-267 and the point-to-point twin) --------
// The adaptors hold the reference constructors' inputs; the ICP objects hand them to cb_icp_set_features, whose device
// search works on [p], [p, w_n n], [p, w_c c] or [p, w_n n, w_c c] exactly as the kd-tree over the adaptors would
// (DESIGN §4.16). Only the 3-D float instances exist, like every other class here.

// IdentityWeightEvaluator / DistanceEvaluator (core/common_pair_evaluators.hpp:13-27, :82): the correspondence value is
// the squared feature distance itself (the only distance evaluator the device search implements)
template <typename ValueT = float, typename WeightT = ValueT>
class DistanceEvaluator {
public:
  using InputScalar = ValueT;
  using OutputScalar = WeightT;
  WeightT operator()(ValueT dist) const { return (WeightT)dist; }
  WeightT operator()(size_t, size_t, ValueT dist) const { return (WeightT)dist; }
};

namespace b200 {
// D x N column-major feature matrix, the pre-assembled form of the adaptors' first constructor
template <int D>
class ConstFeatureMatrixMap {
public:
  ConstFeatureMatrixMap(const float* data = nullptr, size_t n = 0) : p_(data), n_(n) {}
  ConstFeatureMatrixMap(const std::vector<float>& s) : p_(s.data()), n_(s.size() / D) {}
#ifdef CILANTRO_B200_HAS_EIGEN
  ConstFeatureMatrixMap(const Eigen::Matrix<float, D, Eigen::Dynamic>& m) : p_(m.data()), n_((size_t)m.cols()) {}
#endif
  const float* data() const { return p_; }
  size_t cols() const { return n_; }

private:
  const float* p_;
  size_t n_;
};

template <int kKind>
class FeaturesAdaptor3f {
public:
  using Scalar = float;
  enum { FeatureDimension = kKind == CB_FEATURES_POINT_NORMAL_COLOR ? 9 : (kKind == CB_FEATURES_POINT ? 3 : 6) };
  static constexpr int b200_kind() { return kKind; }

  // pre-assembled [p; tails] (tails already weighted)
  FeaturesAdaptor3f(const ConstFeatureMatrixMap<FeatureDimension>& data) : points_(3, data.cols()) {
    constexpr bool nrm = kKind == CB_FEATURES_POINT_NORMAL || kKind == CB_FEATURES_POINT_NORMAL_COLOR;
    constexpr bool col = kKind == CB_FEATURES_POINT_COLOR || kKind == CB_FEATURES_POINT_NORMAL_COLOR;
    if (nrm) normals_.resize(3, data.cols());
    if (col) colors_.resize(3, data.cols());
    for (size_t i = 0; i < data.cols(); i++)
      for (int k = 0; k < 3; k++) {
        const float* c = data.data() + (size_t)FeatureDimension * i;
        points_(k, i) = c[k];
        if (nrm) normals_(k, i) = c[3 + k];
        if (col) colors_(k, i) = c[(nrm ? 6 : 3) + k];
      }
  }
  // PointFeaturesAdaptor (:13-17)
  template <int K = kKind, typename std::enable_if<K == CB_FEATURES_POINT, int>::type = 0>
  FeaturesAdaptor3f(const ConstVectorSetMatrixMap3f& points) : points_(copy(points)) {}
  // PointNormalFeaturesAdaptor (:75-83) / PointColorFeaturesAdaptor (:175-183)
  template <int K = kKind, typename std::enable_if<K == CB_FEATURES_POINT_NORMAL || K == CB_FEATURES_POINT_COLOR, int>::type = 0>
  FeaturesAdaptor3f(const ConstVectorSetMatrixMap3f& points, const ConstVectorSetMatrixMap3f& tail, float weight)
      : points_(copy(points)) {
    (K == CB_FEATURES_POINT_NORMAL ? normals_ : colors_) = copy(tail);
    (K == CB_FEATURES_POINT_NORMAL ? w_n_ : w_c_) = weight;
  }
  // PointNormalColorFeaturesAdaptor (:248-259)
  template <int K = kKind, typename std::enable_if<K == CB_FEATURES_POINT_NORMAL_COLOR, int>::type = 0>
  FeaturesAdaptor3f(const ConstVectorSetMatrixMap3f& points, const ConstVectorSetMatrixMap3f& normals,
                    const ConstVectorSetMatrixMap3f& colors, float normal_weight, float color_weight)
      : points_(copy(points)), normals_(copy(normals)), colors_(copy(colors)), w_n_(normal_weight), w_c_(color_weight) {}

  size_t b200_size() const { return points_.cols(); }
  const float* b200_normals() const { return normals_.cols() ? normals_.data() : nullptr; }
  const float* b200_colors() const { return colors_.cols() ? colors_.data() : nullptr; }
  float b200_normal_weight() const { return w_n_; }
  float b200_color_weight() const { return w_c_; }

private:
  static VectorSet3f copy(const ConstVectorSetMatrixMap3f& m) {
    VectorSet3f s(3, m.cols());
    if (m.cols()) std::memcpy(s.data(), m.data(), 3 * m.cols() * sizeof(float));
    return s;
  }
  VectorSet3f points_, normals_, colors_;
  float w_n_ = 1.f, w_c_ = 1.f;  // the pre-assembled form carries weighted tails: 1 * x = x exactly
};
}  // namespace b200

using PointFeaturesAdaptor3f = b200::FeaturesAdaptor3f<CB_FEATURES_POINT>;
using PointNormalFeaturesAdaptor3f = b200::FeaturesAdaptor3f<CB_FEATURES_POINT_NORMAL>;
using PointColorFeaturesAdaptor3f = b200::FeaturesAdaptor3f<CB_FEATURES_POINT_COLOR>;
using PointNormalColorFeaturesAdaptor3f = b200::FeaturesAdaptor3f<CB_FEATURES_POINT_NORMAL_COLOR>;

// CorrespondenceSearchKDTree<SearchFeatureAdaptorT> (correspondence_search_kd_tree.hpp:41-51, the 3-argument form): the
// engine's fluent setters, and the two feature adaptors the ICP object searches on. The adaptors are held by reference,
// as the reference does.
template <class SearchFeatureAdaptorT, class EvaluatorT = DistanceEvaluator<float, float>>
class CorrespondenceSearchKDTree : public CorrespondenceSearchEngineB200 {
public:
  using SearchResult = CorrespondenceSet<float, size_t>;
  CorrespondenceSearchKDTree(SearchFeatureAdaptorT& dst_features, SearchFeatureAdaptorT& src_features,
                             EvaluatorT& evaluator)
      : dst_(dst_features), src_(src_features), eval_(evaluator) {}
  SearchFeatureAdaptorT& b200_dst_features() { return dst_; }
  SearchFeatureAdaptorT& b200_src_features() { return src_; }
  EvaluatorT& evaluator() { return eval_; }
  // after the ICP's estimate(), as the reference's engine holds them
  const SearchResult& getCorrespondences() const { return feat_corr_; }
  void b200_set_correspondences(const SearchResult& c) { feat_corr_ = c; }

private:
  SearchFeatureAdaptorT& dst_;
  SearchFeatureAdaptorT& src_;
  EvaluatorT& eval_;
  SearchResult feat_corr_;
};

namespace b200 {
// The engine-templated ICP classes: the reference's constructor order, the engine's settings and features read at every
// estimate().
template <class Engine, class Base>
class EngineRigidICP3f : public Base {
public:
  template <class... Args>
  EngineRigidICP3f(Engine& engine, Args&&... args) : Base(std::forward<Args>(args)...), engine_(engine) {}
  Engine& correspondenceSearchEngine() { return engine_; }
  const Engine& correspondenceSearchEngine() const { return engine_; }
  EngineRigidICP3f& estimate() {
    auto& dst = engine_.b200_dst_features();
    auto& src = engine_.b200_src_features();
    if (dst.b200_size() != n_dst_ || src.b200_size() != n_src_)
      throw std::invalid_argument("cilantro_b200: the feature adaptors' sizes differ from the ICP's point sets");
    check(cb_icp_set_features(this->b200_icp(), dst.b200_kind(), dst.b200_normals(), dst.b200_colors(),
                              src.b200_normals(), src.b200_colors(), dst.b200_normal_weight(), dst.b200_color_weight()),
          "cb_icp_set_features");
    Base::correspondenceSearchEngine() = static_cast<const CorrespondenceSearchEngineB200&>(engine_);
    Base::estimate();
    return *this;
  }
  EngineRigidICP3f& estimate(size_t max_iter, float conv_tol) {
    this->setMaxNumberOfIterations(max_iter);
    this->setConvergenceTolerance(conv_tol);
    return estimate();
  }
  const CorrespondenceSet<float, size_t>& getCorrespondences() {
    engine_.b200_set_correspondences(Base::getCorrespondences());
    return engine_.getCorrespondences();
  }

private:
  Engine& engine_;

protected:
  size_t n_dst_ = 0, n_src_ = 0;
};
}  // namespace b200

// PointToPointMetricRigidTransformICP3f<Engine> (icp_single_transform_point_to_point_metric.hpp:21-28, :96-98)
template <class CorrespondenceSearchEngineT>
class PointToPointMetricRigidTransformICP3f
    : public b200::EngineRigidICP3f<CorrespondenceSearchEngineT, SimpleRigidICP3fB200<CB_ICP_POINT_TO_POINT>> {
  using Base = b200::EngineRigidICP3f<CorrespondenceSearchEngineT, SimpleRigidICP3fB200<CB_ICP_POINT_TO_POINT>>;

public:
  PointToPointMetricRigidTransformICP3f(const ConstVectorSetMatrixMap3f& dst, const ConstVectorSetMatrixMap3f& src,
                                        CorrespondenceSearchEngineT& corr_engine)
      : Base(corr_engine, dst, src) {
    this->n_dst_ = dst.cols();
    this->n_src_ = src.cols();
  }
};

// CombinedMetricRigidTransformICP3f<Engine, PtEval, PlEval> (icp_single_transform_combined_metric.hpp:33-40, :63-70;
// icp_common_instances.hpp:262-267)
template <class CorrespondenceSearchEngineT,
          class PointToPointCorrWeightEvaluatorT = UnityWeightEvaluator<float, float>,
          class PointToPlaneCorrWeightEvaluatorT = UnityWeightEvaluator<float, float>>
class CombinedMetricRigidTransformICP3f
    : public b200::EngineRigidICP3f<CorrespondenceSearchEngineT,
                                    CombinedMetricRigidICP3f<PointToPointCorrWeightEvaluatorT, PointToPlaneCorrWeightEvaluatorT>> {
  using Base = b200::EngineRigidICP3f<CorrespondenceSearchEngineT,
                                      CombinedMetricRigidICP3f<PointToPointCorrWeightEvaluatorT, PointToPlaneCorrWeightEvaluatorT>>;

public:
  CombinedMetricRigidTransformICP3f(const ConstVectorSetMatrixMap3f& dst_p, const ConstVectorSetMatrixMap3f& dst_n,
                                    const ConstVectorSetMatrixMap3f& src_p, CorrespondenceSearchEngineT& corr_engine,
                                    PointToPointCorrWeightEvaluatorT& point_corr_eval,
                                    PointToPlaneCorrWeightEvaluatorT& plane_corr_eval)
      : Base(corr_engine, dst_p, dst_n, src_p, point_corr_eval, plane_corr_eval) {
    this->n_dst_ = dst_p.cols();
    this->n_src_ = src_p.cols();
  }
  CombinedMetricRigidTransformICP3f(const ConstVectorSetMatrixMap3f& dst_p, const ConstVectorSetMatrixMap3f& dst_n,
                                    const ConstVectorSetMatrixMap3f& src_p, const ConstVectorSetMatrixMap3f& src_n,
                                    CorrespondenceSearchEngineT& corr_engine,
                                    PointToPointCorrWeightEvaluatorT& point_corr_eval,
                                    PointToPlaneCorrWeightEvaluatorT& plane_corr_eval)
      : Base(corr_engine, dst_p, dst_n, src_p, src_n, point_corr_eval, plane_corr_eval) {
    this->n_dst_ = dst_p.cols();
    this->n_src_ = src_p.cols();
  }
};

// transformPoints(tform, in, out) — core/space_transformations.hpp:203-216
inline void transformPoints(const RigidTransform3f& tform, const ConstVectorSetMatrixMap3f& points, VectorSet3f& result) {
  result.resize(3, points.cols());
  b200::check(cb_transform_points(b200::Context::get(), tform.data(), points.data(), points.cols(), result.data()),
              "cb_transform_points");
}

// ---- TransformSet<RigidTransform3f> (core/space_transformations.hpp:60-136) -----------------------------------
// One transform per point: what the warp-field ICP estimates. Only the surface its callers use.
template <class TransformT>
class TransformSet : public std::vector<TransformT> {
public:
  using std::vector<TransformT>::vector;
  TransformSet& setIdentity() {
    for (auto& t : *this) t.setIdentity();
    return *this;
  }
};
using RigidTransformSet3f = TransformSet<RigidTransform3f>;

// transformPoints(tforms, in, out) (core/space_transformations.hpp:195-223): point i by transform i, in the device's
// float order ((R_r0 x + (R_r1 y + R_r2 z)) + t_r, RigidTransform3f::operator*)
inline void transformPoints(const TransformSet<RigidTransform3f>& tforms, const ConstVectorSetMatrixMap3f& points,
                            VectorSet3f& result) {
  if (tforms.size() != points.cols()) throw std::runtime_error("transformPoints: one transform per point expected");
  result.resize(3, points.cols());
  for (size_t i = 0; i < points.cols(); i++) result.setCol(i, tforms[i] * points.col(i));
}

namespace b200 {
// The surface both warp-field ICP drop-ins share: IterativeClosestPointBase (registration/icp_base.hpp:40-106) and
// CombinedMetric*WarpFieldICP over their cb_warp_params, the correspondence engine and evaluators, the dst/src cloud
// pair and the last estimate's correspondences. Setters return Derived, so calls chain as in the reference. Result is
// the C result record (iterations, last_delta, cg_iterations); the transforms are one per unknown block.
template <class Derived, class Result>
class WarpFieldICP {
public:
  using Transform = TransformSet<RigidTransform3f>;
  using PointToPointCorrespondenceWeightEvaluator = UnityWeightEvaluator<float, float>;
  using PointToPlaneCorrespondenceWeightEvaluator = UnityWeightEvaluator<float, float>;
  using RegularizationWeightEvaluator = RBFKernelWeightEvaluator<float, float, true>;

  WarpFieldICP(const WarpFieldICP&) = delete;
  WarpFieldICP& operator=(const WarpFieldICP&) = delete;

  CorrespondenceSearchEngineB200& correspondenceSearchEngine() { return engine_; }
  PointToPointCorrespondenceWeightEvaluator& pointToPointCorrespondenceWeightEvaluator() { return pt_eval_; }
  PointToPlaneCorrespondenceWeightEvaluator& pointToPlaneCorrespondenceWeightEvaluator() { return pl_eval_; }
  RegularizationWeightEvaluator& regularizationWeightEvaluator() { return reg_eval_; }

  // IterativeClosestPointBase surface
  size_t getMaxNumberOfIterations() const { return (size_t)p_.max_iter; }
  Derived& setMaxNumberOfIterations(size_t n) {
    p_.max_iter = (int32_t)n;
    return self();
  }
  float getConvergenceTolerance() const { return p_.tol; }
  Derived& setConvergenceTolerance(float tol) {
    p_.tol = tol;
    return self();
  }
  const Transform& getInitialTransform() const { return transform_init_; }
  Transform& initialTransform() { return transform_init_; }
  Derived& setInitialTransform(const Transform& T) {
    transform_init_ = T;
    return self();
  }
  size_t getNumberOfPerformedIterations() const { return (size_t)res_.iterations; }
  float getLastUpdateNorm() const { return res_.last_delta; }
  bool hasConverged() const { return res_.last_delta < p_.tol; }  // icp_base.hpp:106
  const Transform& getTransform() const { return transform_; }
  Derived& estimate(size_t max_iter, float conv_tol) {
    p_.max_iter = (int32_t)max_iter;
    p_.tol = conv_tol;
    return self().estimate();
  }

  // CombinedMetric*WarpFieldICP surface
  float getPointToPointMetricWeight() const { return p_.w_pt; }
  Derived& setPointToPointMetricWeight(float w) {
    p_.w_pt = w;
    return self();
  }
  float getPointToPlaneMetricWeight() const { return p_.w_pl; }
  Derived& setPointToPlaneMetricWeight(float w) {
    p_.w_pl = w;
    return self();
  }
  float getStiffnessRegularizationWeight() const { return p_.stiffness; }
  Derived& setStiffnessRegularizationWeight(float w) {
    p_.stiffness = w;
    return self();
  }
  size_t getMaxNumberOfGaussNewtonIterations() const { return (size_t)p_.max_gn_iter; }
  Derived& setMaxNumberOfGaussNewtonIterations(size_t n) {
    p_.max_gn_iter = n;
    return self();
  }
  float getGaussNewtonConvergenceTolerance() const { return p_.gn_tol; }
  Derived& setGaussNewtonConvergenceTolerance(float tol) {
    p_.gn_tol = tol;
    return self();
  }
  size_t getMaxNumberOfConjugateGradientIterations() const { return (size_t)p_.max_cg_iter; }
  Derived& setMaxNumberOfConjugateGradientIterations(size_t n) {
    p_.max_cg_iter = n;
    return self();
  }
  float getConjugateGradientConvergenceTolerance() const { return p_.cg_tol; }
  Derived& setConjugateGradientConvergenceTolerance(float tol) {
    p_.cg_tol = tol;
    return self();
  }
  float getHuberLossBoundary() const { return p_.huber; }
  Derived& setHuberLossBoundary(float huber_boundary) {
    p_.huber = huber_boundary;
    return self();
  }

  uint64_t getNumberOfConjugateGradientIterations() const { return res_.cg_iterations; }  // over the last estimate()

protected:
  // p: the derived class's cb_warp_params (filled by it); n_blocks: the transforms' count
  WarpFieldICP(cb_warp_params& p, const ConstVectorSetMatrixMap3f& dst_p, const ConstVectorSetMatrixMap3f& dst_n,
               const ConstVectorSetMatrixMap3f& src_p, size_t n_blocks)
      : n_src_(src_p.cols()), p_(p) {
    const float* dn = (dst_n.cols() == dst_p.cols() && dst_p.cols() > 0) ? dst_n.data() : nullptr;
    check(cb_cloud_create_pair(Context::get(), dst_p.data(), dn, dst_p.cols(), 0, src_p.data(), nullptr,
                               src_p.cols(), 0, &dst_.h, &src_.h),
          "cb_cloud_create_pair");
    std::memset(&res_, 0, sizeof(res_));
    res_.last_delta = std::numeric_limits<float>::infinity();
    transform_init_.assign(n_blocks, RigidTransform3f());
    transform_.assign(n_blocks, RigidTransform3f());
  }
  ~WarpFieldICP() = default;

  Derived& self() { return static_cast<Derived&>(*this); }

  // neighbourhood lists -> the (offsets, index, value) CSR of the C entries
  template <typename IndexT>
  static void csr(const std::vector<NeighborSet<float, IndexT>>& lists, std::vector<uint64_t>& off,
                  std::vector<int64_t>& idx, std::vector<float>& val) {
    off.assign(lists.size() + 1, 0);
    for (size_t j = 0; j < lists.size(); j++) {
      for (const auto& nb : lists[j]) {
        idx.push_back(static_cast<int64_t>(nb.index));
        val.push_back(nb.value);
      }
      off[j + 1] = idx.size();
    }
  }

  // the engine's and the regularisation evaluator's settings into p_
  void fill() {
    cb_icp_params e;
    cb_icp_default_params(&e);
    engine_.fill(e);
    p_.max_d2 = e.max_d2;
    p_.search_dir = e.search_dir;
    p_.inlier_fraction = e.inlier_fraction;
    p_.require_reciprocal = e.require_reciprocal;
    p_.one_to_one = e.one_to_one;
    p_.reg_coeff = reg_eval_.b200_coeff();
  }

  // correspondenceSearchEngine().getCorrespondences() after estimate(): the last iteration's list, read through the
  // object's cb_*_correspondences entry
  template <class Handle>
  const CorrespondenceSet<float, size_t>& correspondences(int (*entry)(Handle*, uint64_t*, uint64_t*, float*, size_t*),
                                                          Handle* icp, const char* what) {
    if (!corr_fresh_) {
      std::vector<uint64_t> a(n_src_), b(n_src_);
      std::vector<float> v(n_src_);
      size_t cnt = 0;
      check(entry(icp, a.data(), b.data(), v.data(), &cnt), what);
      corr_.resize(cnt);
      for (size_t i = 0; i < cnt; i++) corr_[i] = {(size_t)a[i], (size_t)b[i], v[i]};
      corr_fresh_ = true;
    }
    return corr_;
  }

  size_t n_src_;
  CloudHandle dst_, src_;
  cb_warp_params& p_;
  Result res_;
  Transform transform_init_, transform_;
  CorrespondenceSearchEngineB200 engine_;
  PointToPointCorrespondenceWeightEvaluator pt_eval_;
  PointToPlaneCorrespondenceWeightEvaluator pl_eval_;
  RegularizationWeightEvaluator reg_eval_;  // sigma 1 (common_pair_evaluators.hpp:51)
  CorrespondenceSet<float, size_t> corr_;
  bool corr_fresh_ = false;
};
}  // namespace b200

// ---- SimpleCombinedMetricDenseRigidWarpFieldICP3f (registration/icp_common_instances.hpp:99-144, 284-285) ----------
// CombinedMetricDenseWarpFieldICP<RigidTransform<float,3>> (icp_warp_field_combined_metric_dense.hpp) with the Simple
// instance's evaluators (unity data-term weights, RBFKernelWeightEvaluator<float, float, true> regularisation weights)
// on cb_warp_icp_* (DESIGN §4.13). The correspondence engine takes the default settings only; another search
// direction, reciprocity, one-to-one or fraction makes estimate() throw (CB_ERR_UNSUPPORTED).
class SimpleCombinedMetricDenseRigidWarpFieldICP3f
    : public b200::WarpFieldICP<SimpleCombinedMetricDenseRigidWarpFieldICP3f, cb_warp_result> {
public:
  using WarpFieldICP::estimate;

  // regularization_neighborhoods: one list per neighbourhood, N[0] the centre (what KDTree3f<>::search returns)
  template <typename IndexT>
  SimpleCombinedMetricDenseRigidWarpFieldICP3f(const ConstVectorSetMatrixMap3f& dst_p,
                                               const ConstVectorSetMatrixMap3f& dst_n,
                                               const ConstVectorSetMatrixMap3f& src_p,
                                               const std::vector<NeighborSet<float, IndexT>>& regularization_neighborhoods)
      : WarpFieldICP(prm_, dst_p, dst_n, src_p, src_p.cols()) {
    std::vector<uint64_t> off;
    std::vector<int64_t> idx;
    std::vector<float> val;
    csr(regularization_neighborhoods, off, idx, val);
    b200::check(cb_warp_icp_create(b200::Context::get(), dst_.h, src_.h, off.data(), idx.data(), val.data(),
                                   regularization_neighborhoods.size(), &icp_),
                "cb_warp_icp_create");
    cb_warp_default_params(&prm_);
  }
  ~SimpleCombinedMetricDenseRigidWarpFieldICP3f() {
    if (icp_) cb_warp_icp_destroy(icp_);
  }

  SimpleCombinedMetricDenseRigidWarpFieldICP3f& estimate() {
    if (transform_init_.size() != n_src_) throw std::runtime_error("initial transform: one transform per source point expected");
    fill();
    std::vector<float> T_in(12 * n_src_), T_out(12 * n_src_);
    for (size_t i = 0; i < n_src_; i++) std::memcpy(&T_in[12 * i], transform_init_[i].data(), 12 * sizeof(float));
    b200::check(cb_warp_icp_estimate(icp_, &prm_, T_in.data(), T_out.data(), &res_), "cb_warp_icp_estimate");
    transform_.resize(n_src_);
    for (size_t i = 0; i < n_src_; i++) transform_[i] = RigidTransform3f(&T_out[12 * i]);
    corr_fresh_ = false;
    return *this;
  }

  // getResiduals() -> computeResiduals() (icp_warp_field_combined_metric_dense.hpp:216-236): 1 x N_src
  std::vector<float> getResiduals() {
    fill();
    std::vector<float> T(12 * n_src_), r(n_src_);
    for (size_t i = 0; i < n_src_ && i < transform_.size(); i++) std::memcpy(&T[12 * i], transform_[i].data(), 12 * sizeof(float));
    b200::check(cb_warp_icp_residuals(icp_, &prm_, T.data(), r.data()), "cb_warp_icp_residuals");
    return r;
  }

  const CorrespondenceSet<float, size_t>& getCorrespondences() {
    return correspondences(cb_warp_icp_correspondences, icp_, "cb_warp_icp_correspondences");
  }

  double getLastEstimateDeviceMilliseconds() const { return res_.gpu_ms_search + res_.gpu_ms_solve; }

private:
  cb_warp_icp* icp_ = nullptr;
  cb_warp_params prm_;
};

// ---- SimpleCombinedMetricSparseRigidWarpFieldICP3f (registration/icp_common_instances.hpp:146-199, 313-314) ---------
// CombinedMetricSparseWarpFieldICP<RigidTransform<float,3>> (icp_warp_field_combined_metric_sparse.hpp) with the Simple
// instance's evaluators (unity data-term weights, RBFKernelWeightEvaluator<float, float, true> control and
// regularisation weights) on cb_sparse_warp_icp_* (DESIGN §4.14). getTransform() holds one transform per control
// node, getDenseWarpField() one per source point. The correspondence engine takes the default settings only.
class SimpleCombinedMetricSparseRigidWarpFieldICP3f
    : public b200::WarpFieldICP<SimpleCombinedMetricSparseRigidWarpFieldICP3f, cb_sparse_warp_result> {
public:
  using ControlWeightEvaluator = RBFKernelWeightEvaluator<float, float, true>;
  using WarpFieldICP::estimate;

  // src_to_control_nn: one list of (node, squared distance) per source point; regularization_nn: one list per node
  // neighbourhood, N[0] the centre (what KDTree<float, 3>::search over the nodes returns)
  template <typename IndexT, typename RegIndexT>
  SimpleCombinedMetricSparseRigidWarpFieldICP3f(const ConstVectorSetMatrixMap3f& dst_p,
                                                const ConstVectorSetMatrixMap3f& dst_n,
                                                const ConstVectorSetMatrixMap3f& src_p,
                                                const std::vector<NeighborSet<float, IndexT>>& src_to_control_nn,
                                                size_t num_control_nodes,
                                                const std::vector<NeighborSet<float, RegIndexT>>& regularization_nn)
      : WarpFieldICP(prm_.base, dst_p, dst_n, src_p, num_control_nodes), n_ctrl_(num_control_nodes) {
    std::vector<uint64_t> coff, roff;
    std::vector<int64_t> cidx, ridx;
    std::vector<float> cval, rval;
    csr(src_to_control_nn, coff, cidx, cval);
    csr(regularization_nn, roff, ridx, rval);
    b200::check(cb_sparse_warp_icp_create(b200::Context::get(), dst_.h, src_.h, coff.data(), cidx.data(), cval.data(),
                                          src_to_control_nn.size(), n_ctrl_, roff.data(), ridx.data(), rval.data(),
                                          regularization_nn.size(), &icp_),
                "cb_sparse_warp_icp_create");
    cb_sparse_warp_default_params(&prm_);
    transform_dense_.assign(n_src_, RigidTransform3f());
  }
  ~SimpleCombinedMetricSparseRigidWarpFieldICP3f() {
    if (icp_) cb_sparse_warp_icp_destroy(icp_);
  }

  ControlWeightEvaluator& controlWeightEvaluator() { return ctrl_eval_; }
  const Transform& getDenseWarpField() const { return transform_dense_; }

  SimpleCombinedMetricSparseRigidWarpFieldICP3f& estimate() {
    if (transform_init_.size() != n_ctrl_) throw std::runtime_error("initial transform: one transform per control node expected");
    fill();
    std::vector<float> T_in(12 * n_ctrl_), T_out(12 * n_ctrl_), T_dense(12 * n_src_);
    for (size_t j = 0; j < n_ctrl_; j++) std::memcpy(&T_in[12 * j], transform_init_[j].data(), 12 * sizeof(float));
    b200::check(cb_sparse_warp_icp_estimate(icp_, &prm_, T_in.data(), T_out.data(), T_dense.data(), &res_),
                "cb_sparse_warp_icp_estimate");
    for (size_t j = 0; j < n_ctrl_; j++) transform_[j] = RigidTransform3f(&T_out[12 * j]);
    for (size_t i = 0; i < n_src_; i++) transform_dense_[i] = RigidTransform3f(&T_dense[12 * i]);
    corr_fresh_ = false;
    return *this;
  }

  // getResiduals() -> computeResiduals() (icp_warp_field_combined_metric_sparse.hpp:243-263) on the dense field
  std::vector<float> getResiduals() {
    fill();
    std::vector<float> T(12 * n_src_), r(n_src_);
    for (size_t i = 0; i < n_src_; i++) std::memcpy(&T[12 * i], transform_dense_[i].data(), 12 * sizeof(float));
    b200::check(cb_sparse_warp_icp_residuals(icp_, &prm_, T.data(), r.data()), "cb_sparse_warp_icp_residuals");
    return r;
  }

  const CorrespondenceSet<float, size_t>& getCorrespondences() {
    return correspondences(cb_sparse_warp_icp_correspondences, icp_, "cb_sparse_warp_icp_correspondences");
  }

  double getLastEstimateDeviceMilliseconds() const {
    return res_.gpu_ms_search + res_.gpu_ms_resample + res_.gpu_ms_assemble + res_.gpu_ms_cg;
  }

private:
  void fill() {
    WarpFieldICP::fill();
    prm_.ctrl_coeff = ctrl_eval_.b200_coeff();
  }
  size_t n_ctrl_;
  cb_sparse_warp_icp* icp_ = nullptr;
  cb_sparse_warp_params prm_;
  Transform transform_dense_;
  ControlWeightEvaluator ctrl_eval_;  // sigma 1 (common_pair_evaluators.hpp:51)
};

// ---- KMeans3f<> -------------------------------------------------------------------------------------
template <typename PointIndexT = size_t, typename ClusterIndexT = size_t>
class KMeans3f {
public:
  using ClusterToPointIndicesMap = std::vector<std::vector<PointIndexT>>;
  using PointToClusterIndexMap = std::vector<ClusterIndexT>;

  KMeans3f(const ConstVectorSetMatrixMap3f& data) : n_(data.cols()), host_(data), cloud_(data) {}

  KMeans3f& cluster(const ConstVectorSetMatrixMap3f& centroids, size_t max_iter = 100,
                    float tol = std::numeric_limits<float>::epsilon(), bool use_kd_tree = false) {
    (void)use_kd_tree;  // both branches of the reference compute the same assignment; one GPU kernel here
    centroids_.resize(3, centroids.cols());
    std::memcpy(centroids_.data(), centroids.data(), 3 * centroids.cols() * sizeof(float));
    return run(max_iter, tol);
  }
  KMeans3f& cluster(size_t num_clusters, size_t max_iter = 100, float tol = std::numeric_limits<float>::epsilon(),
                    bool use_kd_tree = false, uint32_t seed = b200::random_seed()) {
    (void)use_kd_tree;
    const size_t k = std::max<size_t>(1, std::min(num_clusters, n_));  // kmeans.hpp:34-36
    std::vector<uint64_t> idx(k);
    b200::check(cb_kmeans_seed_indices(n_, k, seed, idx.data()), "cb_kmeans_seed_indices");
    centroids_.resize(3, k);
    for (size_t j = 0; j < k; j++) centroids_.setCol(j, host_.col(idx[j]));
    return run(max_iter, tol);
  }
  const VectorSet3f& getClusterCentroids() const { return centroids_; }
  size_t getNumberOfPerformedIterations() const { return iterations_; }
  const PointToClusterIndexMap& getPointToClusterIndexMap() const { return labels_; }
  const ClusterToPointIndicesMap& getClusterToPointIndicesMap() const { return lists_; }
  size_t getNumberOfClusters() const { return lists_.size(); }
  size_t getNumberOfPoints() const { return labels_.size(); }

private:
  struct std_seed_helper {};
  KMeans3f& run(size_t max_iter, float tol) {
    std::vector<uint64_t> lab(n_);
    cb_kmeans_result r;
    b200::check(cb_kmeans_cluster(b200::Context::get(), cloud_.h, centroids_.data(), centroids_.cols(), max_iter, tol,
                                  lab.data(), &r),
                "cb_kmeans_cluster");
    iterations_ = r.iterations;
    labels_.assign(lab.begin(), lab.end());
    lists_.assign(centroids_.cols(), {});  // clustering_base.hpp:22-32
    for (size_t i = 0; i < labels_.size(); i++)
      if ((size_t)labels_[i] < lists_.size()) lists_[labels_[i]].emplace_back((PointIndexT)i);
    return *this;
  }
  size_t n_;
  ConstVectorSetMatrixMap3f host_;
  b200::CloudHandle cloud_;
  VectorSet3f centroids_;
  size_t iterations_ = 0;
  PointToClusterIndexMap labels_;
  ClusterToPointIndicesMap lists_;
};

// ---- RigidTransformRANSACEstimator3f<> ----------------------------------------------------------------
template <typename IndexT = size_t>
class RigidTransformRANSACEstimator3f {
public:
  using Model = RigidTransform3f;
  using ResidualVector = std::vector<float>;
  using IndexVector = std::vector<IndexT>;

  RigidTransformRANSACEstimator3f(const ConstVectorSetMatrixMap3f& dst, const ConstVectorSetMatrixMap3f& src)
      : n_(dst.cols()), dst_(dst), src_(src) {
    defaults();
  }
  template <class CorrespondencesT>
  RigidTransformRANSACEstimator3f(const ConstVectorSetMatrixMap3f& dst, const ConstVectorSetMatrixMap3f& src,
                                  const CorrespondencesT& corr)
      : n_(corr.size()), dst_g_(gather(dst, corr, true)), src_g_(gather(src, corr, false)), dst_(dst_g_), src_(src_g_) {
    defaults();
  }

  // (dst, src, dst_ind, src_ind): pair k = (dst point dst_ind[k], src point src_ind[k])
  // (model_estimation/ransac_transform_estimator.hpp:46-59)
  template <typename IdxT>
  RigidTransformRANSACEstimator3f(const ConstVectorSetMatrixMap3f& dst, const ConstVectorSetMatrixMap3f& src,
                                  const std::vector<IdxT>& dst_ind, const std::vector<IdxT>& src_ind)
      : n_(dst_ind.size()), dst_g_(gather_ind(dst, dst_ind, dst_ind.size())), src_g_(gather_ind(src, src_ind, dst_ind.size())),
        dst_(dst_g_), src_(src_g_) {
    defaults();
  }

  // RandomSampleConsensusBase setters (model_estimation/ransac_base.hpp:29-62)
  RigidTransformRANSACEstimator3f& setMaxInlierResidual(float t) { thresh_ = t; return *this; }
  RigidTransformRANSACEstimator3f& setTargetInlierCount(size_t c) { target_ = c; return *this; }
  RigidTransformRANSACEstimator3f& setMaxNumberOfIterations(size_t n) { max_iter_ = n; return *this; }
  RigidTransformRANSACEstimator3f& setReEstimationStep(bool b) { re_estimate_ = b; return *this; }
  RigidTransformRANSACEstimator3f& setRandomSeed(uint32_t s) { seed_ = s; return *this; }  // injected (SURVEY F8)
  float getMaxInlierResidual() const { return thresh_; }
  size_t getTargetInlierCount() const { return target_; }
  size_t getMaxNumberOfIterations() const { return max_iter_; }
  bool getReEstimationStep() const { return re_estimate_; }

  RigidTransformRANSACEstimator3f& estimate() {
    cb_ransac_result r;
    std::vector<uint64_t> inl(n_);
    residuals_.resize(n_);
    b200::check(cb_ransac_rigid(b200::Context::get(), dst_.h, src_.h, seed_, target_, max_iter_, thresh_,
                                re_estimate_ ? 1 : 0, &r, inl.data(), residuals_.data()),
                "cb_ransac_rigid");
    model_ = RigidTransform3f(r.T);
    iterations_ = r.iterations;
    inliers_.assign(inl.begin(), inl.begin() + r.num_inliers);
    return *this;
  }
  RigidTransformRANSACEstimator3f& estimate(float max_residual, size_t target_inlier_count, size_t max_iter) {
    thresh_ = max_residual;
    target_ = target_inlier_count;
    max_iter_ = max_iter;
    return estimate();
  }
  const Model& getModel() const { return model_; }
  const ResidualVector& getModelResiduals() const { return residuals_; }
  const IndexVector& getModelInliers() const { return inliers_; }
  bool targetInlierCountAchieved() const { return inliers_.size() >= target_; }
  size_t getNumberOfPerformedIterations() const { return iterations_; }
  size_t getNumberOfInliers() const { return inliers_.size(); }

private:
  void defaults() {  // ransac_transform_estimator.hpp:27
    target_ = n_ / 2 + n_ % 2;
    max_iter_ = 100;
    thresh_ = 0.01f;
    re_estimate_ = true;
    seed_ = b200::random_seed();
  }
  template <class CorrespondencesT>
  static VectorSet3f gather(const ConstVectorSetMatrixMap3f& pts, const CorrespondencesT& corr, bool first) {
    VectorSet3f out(3, corr.size());  // :31-44
    for (size_t i = 0; i < corr.size(); i++) out.setCol(i, pts.col(first ? corr[i].indexInFirst : corr[i].indexInSecond));
    return out;
  }
  template <typename IdxT>
  static VectorSet3f gather_ind(const ConstVectorSetMatrixMap3f& pts, const std::vector<IdxT>& ind, size_t count) {
    VectorSet3f out(3, count);  // :53-58 (the loop runs over dst_ind.size() for both sets)
    for (size_t i = 0; i < count; i++) out.setCol(i, pts.col((size_t)ind[i]));
    return out;
  }
  size_t n_;
  VectorSet3f dst_g_, src_g_;
  b200::CloudHandle dst_, src_;
  size_t target_, max_iter_, iterations_ = 0;
  float thresh_;
  bool re_estimate_;
  uint32_t seed_;
  Model model_;
  ResidualVector residuals_;
  IndexVector inliers_;
};

// ---- PrincipalComponentAnalysis3f -----------------------------------------------------------------------
class PrincipalComponentAnalysis3f {
public:
  PrincipalComponentAnalysis3f(const ConstVectorSetMatrixMap3f& data, bool /*parallel*/ = false) {
    b200::CloudHandle c(data);
    b200::check(cb_pca(b200::Context::get(), c.h, mean_.data(), cov_.data(), evals_.data(), evecs_.data()), "cb_pca");
  }
  // subset constructor (core/principal_component_analysis.hpp:24-30): the listed points only
  template <typename ContainerT, typename = decltype(std::declval<const ContainerT&>().begin())>
  PrincipalComponentAnalysis3f(const ConstVectorSetMatrixMap3f& data, const ContainerT& subset, bool /*parallel*/ = false) {
    std::vector<float> sel;
    for (auto it = subset.begin(); it != subset.end(); ++it) {
      const Vector3f p = data.col((size_t)*it);
      sel.insert(sel.end(), {p[0], p[1], p[2]});
    }
    b200::CloudHandle c(ConstVectorSetMatrixMap3f(sel.data(), sel.size() / 3));
    b200::check(cb_pca(b200::Context::get(), c.h, mean_.data(), cov_.data(), evals_.data(), evecs_.data()), "cb_pca");
  }
  const Vector3f& getDataMean() const { return mean_; }
  const std::array<float, 9>& getDataCovariance() const { return cov_; }  // row-major 3x3
  const Vector3f& getEigenValues() const { return evals_; }               // descending
  const std::array<float, 9>& getEigenVectors() const { return evecs_; }  // row-major, columns = eigenvectors

  // project(points, target_dim) (:46-49): target_dim x N, column-major = eigenvectors.leftCols(target_dim)^T (p - mean).
  // A 3 x k map applied once after the device pass, like the reference's Eigen expression (not part of the hot path).
  std::vector<float> project(const ConstVectorSetMatrixMap3f& points, size_t target_dim) const {
    const size_t k = std::min<size_t>(target_dim, 3), n = points.cols();
    std::vector<float> out(k * n);
    for (size_t i = 0; i < n; i++) {
      const Vector3f p = points.col(i);
      const float c[3] = {p[0] - mean_[0], p[1] - mean_[1], p[2] - mean_[2]};
      for (size_t j = 0; j < k; j++) out[k * i + j] = evecs_[j] * c[0] + evecs_[3 + j] * c[1] + evecs_[6 + j] * c[2];
    }
    return out;
  }
  template <size_t DimOut>
  std::vector<float> project(const ConstVectorSetMatrixMap3f& points) const {  // :51-57
    static_assert(DimOut >= 1 && DimOut <= 3, "projection dimension of a 3-D PCA");
    return project(points, DimOut);
  }
  // reconstruct(points) (:59-70): points is dim_in x N column-major; returns 3 x N = leftCols(dim_in) * points + mean
  VectorSet3f reconstruct(const float* points, size_t dim_in, size_t n) const {
    const size_t k = std::min<size_t>(dim_in, 3);
    VectorSet3f out(3, n);
    for (size_t i = 0; i < n; i++) {
      float q[3] = {mean_[0], mean_[1], mean_[2]};
      for (size_t j = 0; j < k; j++)
        for (int r = 0; r < 3; r++) q[r] += evecs_[3 * r + j] * points[dim_in * i + j];
      out.setCol(i, Vector3f(q[0], q[1], q[2]));
    }
    return out;
  }
  VectorSet3f reconstruct(const std::vector<float>& points, size_t dim_in) const {
    return reconstruct(points.data(), dim_in, dim_in ? points.size() / dim_in : 0);
  }

private:
  Vector3f mean_, evals_;
  std::array<float, 9> cov_{}, evecs_{};
};

// ---- PointCloud3f ------------------------------------------------------------------------------------------
// ---- normal estimation (core/normal_estimation.hpp:11-421) ------------------------------------------
// Same call surface as NormalEstimation<float,3>: neighbourhoods over the cloud itself; radii are
// squared distances; fewer than 3 neighbours -> NaN; view point (default: none, :24-25) orients the
// normals; reference normals (setReferenceNormals, :63-69) take precedence over it (:281-291).
class NormalEstimation3f {
public:
  NormalEstimation3f(const ConstVectorSetMatrixMap3f& points, size_t /*max_leaf_size*/ = 10)
      : n_(points.cols()), points_(points), cloud_(points) {
    const float nan = std::numeric_limits<float>::quiet_NaN();
    view_point_ = Vector3f(nan, nan, nan);
  }
  // from an existing search tree (:30-39): the same points; the device grid is rebuilt for this object
  template <typename IndexT>
  explicit NormalEstimation3f(const KDTree3f<IndexT>& kd_tree) : NormalEstimation3f(kd_tree.getPointsMatrixMap()) {}
  // getNormals* (:71-81 and the Radius / KNNInRadius twins): return by value
  VectorSet3f getNormalsKNN(size_t k) const { return estimateNormalsKNN(k); }
  VectorSet3f getNormalsRadius(float radius) const { return estimateNormalsRadius(radius); }
  VectorSet3f getNormalsKNNInRadius(size_t k, float radius) const { return estimateNormalsKNNInRadius(k, radius); }
  const Vector3f& getViewPoint() const { return view_point_; }
  NormalEstimation3f& setViewPoint(const Vector3f& vp) {  // :52-56
    view_point_ = vp;
    return *this;
  }
  NormalEstimation3f& setReferenceNormals(const ConstVectorSetMatrixMap3f& ref_normals) {  // :63-69
    if (ref_normals.cols() == n_) {  // a copy: the caller may pass the very buffer the result goes to
      ref_normals_.assign(ref_normals.data(), ref_normals.data() + 3 * n_);
      use_ref_ = n_ > 0;
    }
    return *this;
  }
  // kNN (:83-129)
  const NormalEstimation3f& estimateNormalsAndCurvatureKNN(VectorSet3f& normals, std::vector<float>& curvature,
                                                           size_t k) const {
    return run(&normals, &curvature, k, 0.f);
  }
  const NormalEstimation3f& estimateNormalsKNN(VectorSet3f& normals, size_t k) const {
    return run(&normals, nullptr, k, 0.f);
  }
  VectorSet3f estimateNormalsKNN(size_t k) const {
    VectorSet3f n;
    run(&n, nullptr, k, 0.f);
    return n;
  }
  const NormalEstimation3f& estimateCurvatureKNN(std::vector<float>& curvature, size_t k) const {
    return run(nullptr, &curvature, k, 0.f);
  }
  // radius (:131-177)
  const NormalEstimation3f& estimateNormalsAndCurvatureRadius(VectorSet3f& normals, std::vector<float>& curvature,
                                                              float radius) const {
    return run(&normals, &curvature, 0, radius);
  }
  const NormalEstimation3f& estimateNormalsRadius(VectorSet3f& normals, float radius) const {
    return run(&normals, nullptr, 0, radius);
  }
  VectorSet3f estimateNormalsRadius(float radius) const {
    VectorSet3f n;
    run(&n, nullptr, 0, radius);
    return n;
  }
  const NormalEstimation3f& estimateCurvatureRadius(std::vector<float>& curvature, float radius) const {
    return run(nullptr, &curvature, 0, radius);
  }
  // kNN in radius (:179-232)
  const NormalEstimation3f& estimateNormalsAndCurvatureKNNInRadius(VectorSet3f& normals,
                                                                   std::vector<float>& curvature, size_t k,
                                                                   float radius) const {
    return run(&normals, &curvature, k, radius);
  }
  const NormalEstimation3f& estimateNormalsKNNInRadius(VectorSet3f& normals, size_t k, float radius) const {
    return run(&normals, nullptr, k, radius);
  }
  VectorSet3f estimateNormalsKNNInRadius(size_t k, float radius) const {
    VectorSet3f n;
    run(&n, nullptr, k, radius);
    return n;
  }
  const NormalEstimation3f& estimateCurvatureKNNInRadius(std::vector<float>& curvature, size_t k,
                                                         float radius) const {
    return run(nullptr, &curvature, k, radius);
  }

private:
  const NormalEstimation3f& run(VectorSet3f* normals, std::vector<float>* curvature, size_t k, float radius) const {
    if (k > 128) throw std::runtime_error("cilantro_b200: normal estimation supports k <= 128 neighbours");
    if (normals) normals->resize(3, n_);
    if (curvature) curvature->resize(n_);
    if (n_ == 0) return *this;
    const float nan = std::numeric_limits<float>::quiet_NaN();
    if (k == 0 && !(radius > 0.f)) {  // empty neighbourhoods: every sample is below the minimum size
      if (normals) std::fill(normals->data(), normals->data() + 3 * n_, nan);
      if (curvature) std::fill(curvature->begin(), curvature->end(), nan);
      return *this;
    }
    if (use_ref_) {  // re-upload the reference normals: the previous call overwrote the cloud's normals
      ConstVectorSetMatrixMap3f ref(ref_normals_);
      cloud_.reset(points_, &ref);
    }
    b200::check(cb_cloud_estimate_normals(b200::Context::get(), cloud_.h, (int)k, radius, view_point_.data(),
                                          use_ref_ ? 1 : 0, normals ? normals->data() : nullptr,
                                          curvature ? curvature->data() : nullptr, nullptr, nullptr),
                "cb_cloud_estimate_normals");
    return *this;
  }
  size_t n_;
  ConstVectorSetMatrixMap3f points_;
  mutable b200::CloudHandle cloud_;
  Vector3f view_point_;
  std::vector<float> ref_normals_;
  bool use_ref_ = false;
};

// ---- voxel-grid downsampling (core/grid_downsampler.hpp, core/grid_accumulator.hpp) ---------------------
// One implementation behind the four reference class names: the constructor takes the same arguments
// (points [, normals] [, colors], bin_size, parallel); parallel selects the reference's output order
// (true: bins in lexicographic (x, y, z) order, the std::map order of the parallel build; false: in order
// of first occurrence, the serial build). The per-bin sums are always the serial build's (index order).
namespace b200 {
class GridDownsampler {
public:
  GridDownsampler(const ConstVectorSetMatrixMap3f& points, const ConstVectorSetMatrixMap3f* normals,
                  const ConstVectorSetMatrixMap3f* colors, float bin_size, bool parallel)
      : points_(points), normals_(normals ? *normals : ConstVectorSetMatrixMap3f()),
        colors_(colors ? *colors : ConstVectorSetMatrixMap3f()), has_n_(normals != nullptr), has_c_(colors != nullptr),
        bin_size_(bin_size), order_(parallel ? 0 : 1) {}

protected:
  void run(VectorSet3f* ds_points, VectorSet3f* ds_normals, VectorSet3f* ds_colors, size_t min_points_in_bin) const {
    const size_t n = points_.cols();
    VectorSet3f p(3, n), nn(3, has_n_ ? n : 0), cc(3, has_c_ ? n : 0);
    size_t m = 0;
    check(cb_grid_downsample(Context::get(), points_.data(), has_n_ ? normals_.data() : nullptr,
                             has_c_ ? colors_.data() : nullptr, n, bin_size_, min_points_in_bin, order_, p.data(),
                             has_n_ ? nn.data() : nullptr, has_c_ ? cc.data() : nullptr, &m),
          "cb_grid_downsample");
    p.resize(3, m);
    if (ds_points) *ds_points = std::move(p);
    if (ds_normals && has_n_) {
      nn.resize(3, m);
      *ds_normals = std::move(nn);
    }
    if (ds_colors && has_c_) {
      cc.resize(3, m);
      *ds_colors = std::move(cc);
    }
  }
  ConstVectorSetMatrixMap3f points_, normals_, colors_;
  bool has_n_, has_c_;
  float bin_size_;
  int order_;
};
}  // namespace b200

class PointsGridDownsampler3f : public b200::GridDownsampler {  // grid_downsampler.hpp:8-44
public:
  PointsGridDownsampler3f(const ConstVectorSetMatrixMap3f& points, float bin_size, bool parallel = true)
      : GridDownsampler(points, nullptr, nullptr, bin_size, parallel) {}
  const PointsGridDownsampler3f& getDownsampledPoints(VectorSet3f& ds_points, size_t min_points_in_bin = 1) const {
    run(&ds_points, nullptr, nullptr, min_points_in_bin);
    return *this;
  }
  VectorSet3f getDownsampledPoints(size_t min_points_in_bin = 1) const {
    VectorSet3f p;
    run(&p, nullptr, nullptr, min_points_in_bin);
    return p;
  }
};

class PointsNormalsGridDownsampler3f : public b200::GridDownsampler {  // grid_downsampler.hpp:46-132
public:
  PointsNormalsGridDownsampler3f(const ConstVectorSetMatrixMap3f& points, const ConstVectorSetMatrixMap3f& normals,
                                 float bin_size, bool parallel = true)
      : GridDownsampler(points, &normals, nullptr, bin_size, parallel) {}
  const PointsNormalsGridDownsampler3f& getDownsampledPoints(VectorSet3f& p, size_t min_points_in_bin = 1) const {
    run(&p, nullptr, nullptr, min_points_in_bin);
    return *this;
  }
  const PointsNormalsGridDownsampler3f& getDownsampledNormals(VectorSet3f& nn, size_t min_points_in_bin = 1) const {
    run(nullptr, &nn, nullptr, min_points_in_bin);
    return *this;
  }
  const PointsNormalsGridDownsampler3f& getDownsampledPointsNormals(VectorSet3f& p, VectorSet3f& nn,
                                                                    size_t min_points_in_bin = 1) const {
    run(&p, &nn, nullptr, min_points_in_bin);
    return *this;
  }
};

class PointsColorsGridDownsampler3f : public b200::GridDownsampler {  // grid_downsampler.hpp:134-220
public:
  PointsColorsGridDownsampler3f(const ConstVectorSetMatrixMap3f& points, const ConstVectorSetMatrixMap3f& colors,
                                float bin_size, bool parallel = true)
      : GridDownsampler(points, nullptr, &colors, bin_size, parallel) {}
  const PointsColorsGridDownsampler3f& getDownsampledPoints(VectorSet3f& p, size_t min_points_in_bin = 1) const {
    run(&p, nullptr, nullptr, min_points_in_bin);
    return *this;
  }
  const PointsColorsGridDownsampler3f& getDownsampledColors(VectorSet3f& cc, size_t min_points_in_bin = 1) const {
    run(nullptr, nullptr, &cc, min_points_in_bin);
    return *this;
  }
  const PointsColorsGridDownsampler3f& getDownsampledPointsColors(VectorSet3f& p, VectorSet3f& cc,
                                                                  size_t min_points_in_bin = 1) const {
    run(&p, nullptr, &cc, min_points_in_bin);
    return *this;
  }
};

class PointsNormalsColorsGridDownsampler3f : public b200::GridDownsampler {  // grid_downsampler.hpp:222-340
public:
  PointsNormalsColorsGridDownsampler3f(const ConstVectorSetMatrixMap3f& points,
                                       const ConstVectorSetMatrixMap3f& normals,
                                       const ConstVectorSetMatrixMap3f& colors, float bin_size, bool parallel = true)
      : GridDownsampler(points, &normals, &colors, bin_size, parallel) {}
  const PointsNormalsColorsGridDownsampler3f& getDownsampledPoints(VectorSet3f& p, size_t min_points_in_bin = 1) const {
    run(&p, nullptr, nullptr, min_points_in_bin);
    return *this;
  }
  const PointsNormalsColorsGridDownsampler3f& getDownsampledNormals(VectorSet3f& nn,
                                                                    size_t min_points_in_bin = 1) const {
    run(nullptr, &nn, nullptr, min_points_in_bin);
    return *this;
  }
  const PointsNormalsColorsGridDownsampler3f& getDownsampledColors(VectorSet3f& cc, size_t min_points_in_bin = 1) const {
    run(nullptr, nullptr, &cc, min_points_in_bin);
    return *this;
  }
  const PointsNormalsColorsGridDownsampler3f& getDownsampledPointsNormalsColors(VectorSet3f& p, VectorSet3f& nn,
                                                                                VectorSet3f& cc,
                                                                                size_t min_points_in_bin = 1) const {
    run(&p, &nn, &cc, min_points_in_bin);
    return *this;
  }
};

struct PointCloud3f {
  VectorSet3f points, normals, colors;
  PointCloud3f() = default;
  // PLY passthrough (utilities/point_cloud.hpp:118-121, :502-543; b200_ply.hpp)
  explicit PointCloud3f(const std::string& file_name) { fromPLYFile(file_name); }
  // the points listed in `indices` (negate: every other point), sorted and without duplicates, with their normals
  // and colours (utilities/point_cloud.hpp:32-81). The reference leaves the points uninitialised when the cloud has
  // neither normals nor colours; they are copied here in every case.
  template <typename IndexT>
  PointCloud3f(const PointCloud3f& cloud, const std::vector<IndexT>& indices, bool negate = false) {
    std::set<IndexT> keep;
    if (negate) {
      const std::set<IndexT> drop(indices.begin(), indices.end());
      for (size_t i = 0; i < cloud.size(); i++)
        if (!drop.count(static_cast<IndexT>(i))) keep.insert(static_cast<IndexT>(i));
    } else {
      keep.insert(indices.begin(), indices.end());
    }
    const bool has_n = cloud.hasNormals(), has_c = cloud.hasColors();
    points.resize(3, keep.size());
    if (has_n) normals.resize(3, keep.size());
    if (has_c) colors.resize(3, keep.size());
    size_t k = 0;
    for (IndexT i : keep) {
      points.setCol(k, cloud.points.col((size_t)i));
      if (has_n) normals.setCol(k, cloud.normals.col((size_t)i));
      if (has_c) colors.setCol(k, cloud.colors.col((size_t)i));
      k++;
    }
  }
  // remove(indices) (utilities/point_cloud.hpp:154-199): each removed point takes the place of the last kept one, so
  // the order of the survivors is the reference's, not the original order
  template <typename IndexT>
  PointCloud3f& remove(const std::vector<IndexT>& indices) {
    if (indices.empty()) return *this;
    const std::set<IndexT> drop(indices.begin(), indices.end());
    if (drop.size() >= size()) return clear();
    size_t valid = size() - 1;
    while (drop.count(static_cast<IndexT>(valid))) valid--;
    const bool has_n = hasNormals(), has_c = hasColors();
    auto swap_cols = [](VectorSet3f& m, size_t a, size_t b) {
      const Vector3f t = m.col(a);
      m.setCol(a, m.col(b));
      m.setCol(b, t);
    };
    for (auto it = drop.begin(); it != drop.end() && (size_t)*it < valid; ++it) {
      swap_cols(points, (size_t)*it, valid);
      if (has_n) swap_cols(normals, (size_t)*it, valid);
      if (has_c) swap_cols(colors, (size_t)*it, valid);
      valid--;
      while ((size_t)*it < valid && drop.count(static_cast<IndexT>(valid))) valid--;
    }
    const size_t n0 = size(), n1 = valid + 1;
    points.resize(3, n1);
    if (normals.cols() == n0) normals.resize(3, n1);
    if (colors.cols() == n0) colors.resize(3, n1);
    return *this;
  }
  PointCloud3f& fromPLYFile(const std::string& file_name, bool /*preload*/ = true) {
    std::vector<float> p, n, c;
    b200::ply::read(file_name, p, n, c);
    auto assign = [](VectorSet3f& dst, const std::vector<float>& src) {
      dst.resize(3, src.size() / 3);
      if (!src.empty()) std::memcpy(dst.data(), src.data(), src.size() * sizeof(float));
    };
    assign(points, p);
    assign(normals, n);
    assign(colors, c);
    return *this;
  }
  const PointCloud3f& toPLYFile(const std::string& file_name, bool binary = true) const {
    b200::ply::write(file_name, binary, size(), points.data(), hasNormals() ? normals.data() : nullptr,
                     hasColors() ? colors.data() : nullptr);
    return *this;
  }
  PointCloud3f& clear() {  // :131-136
    points.resize(3, 0);
    normals.resize(3, 0);
    colors.resize(3, 0);
    return *this;
  }
  PointCloud3f& append(const PointCloud3f& cloud) {  // :138-152
    const size_t n0 = size(), n1 = cloud.size();
    auto grow = [&](VectorSet3f& dst, const VectorSet3f& src) {
      dst.resize(3, n0 + n1);
      if (n1) std::memcpy(dst.data() + 3 * n0, src.data(), 3 * n1 * sizeof(float));
    };
    const bool keep_n = normals.cols() == n0 && cloud.hasNormals(), keep_c = colors.cols() == n0 && cloud.hasColors();
    grow(points, cloud.points);
    if (keep_n) grow(normals, cloud.normals);
    if (keep_c) grow(colors, cloud.colors);
    return *this;
  }
  // utilities/point_cloud.hpp:246-290
  PointCloud3f& gridDownsample(float bin_size, size_t min_points_in_bin = 1, bool parallel = true) {
    PointCloud3f res = gridDownsampled(bin_size, min_points_in_bin, parallel);
    *this = std::move(res);
    return *this;
  }
  PointCloud3f gridDownsampled(float bin_size, size_t min_points_in_bin = 1, bool parallel = true) const {
    PointCloud3f res;
    if (hasNormals() && hasColors()) {
      PointsNormalsColorsGridDownsampler3f(points, normals, colors, bin_size, parallel)
          .getDownsampledPointsNormalsColors(res.points, res.normals, res.colors, min_points_in_bin);
    } else if (hasNormals()) {
      PointsNormalsGridDownsampler3f(points, normals, bin_size, parallel)
          .getDownsampledPointsNormals(res.points, res.normals, min_points_in_bin);
    } else if (hasColors()) {
      PointsColorsGridDownsampler3f(points, colors, bin_size, parallel)
          .getDownsampledPointsColors(res.points, res.colors, min_points_in_bin);
    } else {
      PointsGridDownsampler3f(points, bin_size, parallel).getDownsampledPoints(res.points, min_points_in_bin);
    }
    return res;
  }
  // utilities/point_cloud.hpp:292-420: view point = origin unless the current normals serve as the
  // reference (use_current_as_ref && hasNormals())
  PointCloud3f& estimateNormalsKNN(size_t k, bool use_current_as_ref = false) {
    normal_estimator(use_current_as_ref).estimateNormalsKNN(normals, k);
    return *this;
  }
  PointCloud3f& estimateNormalsRadius(float radius, bool use_current_as_ref = false) {
    normal_estimator(use_current_as_ref).estimateNormalsRadius(normals, radius);
    return *this;
  }
  PointCloud3f& estimateNormalsKNNInRadius(size_t k, float radius, bool use_current_as_ref = false) {
    normal_estimator(use_current_as_ref).estimateNormalsKNNInRadius(normals, k, radius);
    return *this;
  }
  // overloads taking the caller's search tree (utilities/point_cloud.hpp:311-327 etc.): same result
  template <typename IndexT>
  PointCloud3f& estimateNormalsKNN(const KDTree3f<IndexT>&, size_t k, bool use_current_as_ref = false) {
    return estimateNormalsKNN(k, use_current_as_ref);
  }
  template <typename IndexT>
  PointCloud3f& estimateNormalsRadius(const KDTree3f<IndexT>&, float radius, bool use_current_as_ref = false) {
    return estimateNormalsRadius(radius, use_current_as_ref);
  }
  template <typename IndexT>
  PointCloud3f& estimateNormalsKNNInRadius(const KDTree3f<IndexT>&, size_t k, float radius,
                                           bool use_current_as_ref = false) {
    return estimateNormalsKNNInRadius(k, radius, use_current_as_ref);
  }
  NormalEstimation3f normal_estimator(bool use_current_as_ref) const {
    NormalEstimation3f ne(points);
    if (use_current_as_ref && hasNormals())
      ne.setReferenceNormals(normals);
    else
      ne.setViewPoint(Vector3f(0.f, 0.f, 0.f));
    return ne;
  }
  size_t size() const { return points.cols(); }
  bool hasNormals() const { return size() > 0 && normals.cols() == size(); }
  // removeInvalidNormals() (utilities/point_cloud.hpp:210-219): remove() of the points whose normal is not finite
  PointCloud3f& removeInvalidNormals() {
    if (!hasNormals()) return *this;
    std::vector<size_t> drop;
    for (size_t i = 0; i < normals.cols(); i++) {
      const float* v = normals.data() + 3 * i;
      if (!(std::isfinite(v[0]) && std::isfinite(v[1]) && std::isfinite(v[2]))) drop.push_back(i);
    }
    return remove(drop);
  }
  bool hasColors() const { return size() > 0 && colors.cols() == size(); }
  bool isEmpty() const { return size() == 0; }
  // per-point transforms (a warp field): points by transformPoints(tforms, ...), normals by the linear parts
  PointCloud3f& transform(const TransformSet<RigidTransform3f>& tforms) {
    VectorSet3f out;
    transformPoints(tforms, points, out);
    points = out;
    if (hasNormals()) {
      TransformSet<RigidTransform3f> R = tforms;
      for (auto& t : R)
        for (int r = 0; r < 3; r++) t.translation(r) = 0.f;
      transformPoints(R, normals, out);
      normals = out;
    }
    return *this;
  }
  PointCloud3f transformed(const TransformSet<RigidTransform3f>& tforms) const {
    PointCloud3f res = *this;
    return res.transform(tforms);
  }
  PointCloud3f& transform(const RigidTransform3f& T) {  // utilities/point_cloud.hpp (rigid overload)
    VectorSet3f out;
    transformPoints(T, points, out);
    points = out;
    if (hasNormals()) {
      RigidTransform3f R = T;
      for (int r = 0; r < 3; r++) R.translation(r) = 0.f;
      transformPoints(R, normals, out);
      normals = out;
    }
    return *this;
  }
};

}  // namespace cilantro
