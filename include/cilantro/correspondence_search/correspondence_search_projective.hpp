// Same include path as cilantro's correspondence_search/correspondence_search_projective.hpp: the projective
// correspondence search as the engine of rigid ICP and of the warp-field ICPs, SimpleCombinedMetricRigidProjectiveICP3f
// (registration/icp_common_instances.hpp:223-270), SimpleCombinedMetricDenseRigidWarpFieldProjectiveICP3f and
// SimpleCombinedMetricSparseRigidWarpFieldProjectiveICP3f (:233-245, 298-299, 327-328). The search itself runs on the
// device: estimate() hands the projection to the ICP object (cb_icp_set_projection, cb_warp_icp_set_projection,
// cb_sparse_warp_icp_set_projection; DESIGN §4.21, §4.22), which keeps the index map over the destination on the
// device and rebuilds it only when a projection setter changed. Only the float instance with PointFeaturesAdaptor3f and
// DistanceEvaluator exists; any other ScalarT, evaluation adaptor or evaluator is a compile-time error. Intrinsics are a
// b200::Intrinsics3f (row-major 3 x 3), converted implicitly from an Eigen::Matrix<float, 3, 3> where Eigen is available.
#pragma once
#include <cstdint>
#include <type_traits>

#include "../b200_shims.hpp"
#include "../core/image_point_cloud_conversions.hpp"

namespace cilantro {

template <class ScalarT, class EvaluationFeatureAdaptorT = PointFeaturesAdaptor3f,
          class EvaluatorT = DistanceEvaluator<float, float>, typename IndexT = size_t>
class CorrespondenceSearchProjective {
  static_assert(std::is_same<ScalarT, float>::value, "cilantro_b200 provides the float projective search only");
  static_assert(std::is_same<EvaluationFeatureAdaptorT, PointFeaturesAdaptor3f>::value,
                "cilantro_b200: the projective search evaluates on PointFeaturesAdaptor3f only");
  static_assert(std::is_same<EvaluatorT, DistanceEvaluator<float, float>>::value,
                "cilantro_b200: the projective search's value is the squared distance (DistanceEvaluator) only");
  static_assert(std::is_same<IndexT, size_t>::value, "cilantro_b200: size_t correspondence indices only");

public:
  using Evaluator = EvaluatorT;
  using CorrespondenceScalar = float;
  using CorrespondenceIndex = IndexT;
  using SearchResult = CorrespondenceSet<float, size_t>;

  // :24-39 and :41-57; the defaults are the reference's "Kinect"-like ones
  CorrespondenceSearchProjective(PointFeaturesAdaptor3f& dst_points, PointFeaturesAdaptor3f& src_points,
                                 EvaluatorT& evaluator)
      : dst_(dst_points), src_(src_points), eval_(evaluator) {}
  CorrespondenceSearchProjective(PointFeaturesAdaptor3f& dst_points, PointFeaturesAdaptor3f& src_points,
                                 EvaluationFeatureAdaptorT&, EvaluatorT& evaluator)
      : dst_(dst_points), src_(src_points), eval_(evaluator) {}

  // after the ICP's estimate(): the correspondences of its last iteration
  const SearchResult& getCorrespondences() const { return corr_; }
  Evaluator& evaluator() { return eval_; }

  const b200::Intrinsics3f& getProjectionIntrinsicMatrix() const { return K_; }
  CorrespondenceSearchProjective& setProjectionIntrinsicMatrix(const b200::Intrinsics3f& mat) {
    K_ = mat;
    ++gen_;
    return *this;
  }
  size_t getProjectionImageWidth() const { return w_; }
  CorrespondenceSearchProjective& setProjectionImageWidth(size_t w) {
    w_ = w;
    ++gen_;
    return *this;
  }
  size_t getProjectionImageHeight() const { return h_; }
  CorrespondenceSearchProjective& setProjectionImageHeight(size_t h) {
    h_ = h;
    ++gen_;
    return *this;
  }
  const RigidTransform3f& getProjectionExtrinsicMatrix() const { return E_; }
  CorrespondenceSearchProjective& setProjectionExtrinsicMatrix(const RigidTransform3f& mat) {
    E_ = mat;
    ++gen_;
    return *this;
  }
  float getMaxDistance() const { return settings_.getMaxDistance(); }
  CorrespondenceSearchProjective& setMaxDistance(float dist_thresh) {
    settings_.setMaxDistance(dist_thresh);
    return *this;
  }
  double getInlierFraction() const { return settings_.getInlierFraction(); }
  CorrespondenceSearchProjective& setInlierFraction(double fraction) {
    settings_.setInlierFraction(fraction);
    return *this;
  }

  // estimate() of an ICP object over this engine: (re)attaches the projection through the object's set_projection
  // entry when the object has not taken this state yet (attached: the generation it last took)
  template <class Handle>
  void b200_attach(int (*entry)(Handle*, const float*, size_t, size_t, const float*), Handle* icp, uint64_t& attached,
                   const char* what) {
    if (attached == gen_) return;
    b200::check(entry(icp, K_.m, w_, h_, E_.data()), what);
    attached = gen_;
  }
  // b200::EngineRigidICP3f::estimate()
  void b200_attach(cb_icp* icp, size_t n_dst, size_t n_src, uint64_t& attached) {
    if (dst_.b200_size() != n_dst || src_.b200_size() != n_src)
      throw std::invalid_argument("cilantro_b200: the engine's point adaptors' sizes differ from the ICP's point sets");
    b200_attach(cb_icp_set_projection, icp, attached, "cb_icp_set_projection");
  }
  const CorrespondenceSearchEngineB200& b200_settings() const { return settings_; }
  void b200_set_correspondences(const SearchResult& c) { corr_ = c; }

private:
  PointFeaturesAdaptor3f& dst_;
  PointFeaturesAdaptor3f& src_;
  EvaluatorT& eval_;
  b200::Intrinsics3f K_{528.f, 528.f, 320.f, 240.f};
  size_t w_ = 640, h_ = 480;
  RigidTransform3f E_;                // identity
  CorrespondenceSearchEngineB200 settings_;  // max distance 0.01^2, inlier fraction 1 (the reference's defaults)
  uint64_t gen_ = 1;                  // +1 per projection setter: an ICP object that took an older one re-attaches
  SearchResult corr_;
};

namespace b200 {
// SimpleCombinedMetricICPWrapper's entities (icp_common_instances.hpp:59-73): the adaptors, the evaluator and the engine
// the ICP object owns
struct ProjectiveICPEntities3f {
  ProjectiveICPEntities3f(const ConstVectorSetMatrixMap3f& dst, const ConstVectorSetMatrixMap3f& src)
      : dst_feat_(dst), src_feat_(src), corr_search_(dst_feat_, src_feat_, corr_dist_evaluator_) {}
  PointFeaturesAdaptor3f dst_feat_, src_feat_;
  DistanceEvaluator<float, float> corr_dist_evaluator_;
  CorrespondenceSearchProjective<float> corr_search_;
  UnityWeightEvaluator<float, float> point_corr_weight_eval_, plane_corr_weight_eval_;
};

// The projective engine of a warp-field ICP drop-in, with the adaptors and the evaluator it is built on (see the
// kd-tree engine's WarpEngine in b200_shims.hpp)
template <>
struct WarpEngine<CorrespondenceSearchProjective<float>> {
  WarpEngine(const ConstVectorSetMatrixMap3f& dst, const ConstVectorSetMatrixMap3f& src)
      : dst_feat(dst), src_feat(src), engine(dst_feat, src_feat, dist_eval) {}
  const CorrespondenceSearchEngineB200& settings() const { return engine.b200_settings(); }
  template <class Handle>
  void attach(int (*entry)(Handle*, const float*, size_t, size_t, const float*), Handle* icp, const char* what) {
    engine.b200_attach(entry, icp, attached, what);
  }
  void publish(const CorrespondenceSet<float, size_t>& c) { engine.b200_set_correspondences(c); }
  PointFeaturesAdaptor3f dst_feat, src_feat;
  DistanceEvaluator<float, float> dist_eval;
  CorrespondenceSearchProjective<float> engine;
  uint64_t attached = 0;  // the engine's generation the ICP object last took
};
}  // namespace b200

// SimpleCombinedMetricRigidProjectiveICP3f (icp_common_instances.hpp:223-225, :269-270): the combined metric over the
// projective search, with both of the reference's constructors
class SimpleCombinedMetricRigidProjectiveICP3f : private b200::ProjectiveICPEntities3f,
                                                 public CombinedMetricRigidTransformICP3f<CorrespondenceSearchProjective<float>> {
  using Base = CombinedMetricRigidTransformICP3f<CorrespondenceSearchProjective<float>>;

public:
  SimpleCombinedMetricRigidProjectiveICP3f(const ConstVectorSetMatrixMap3f& dst_points,
                                           const ConstVectorSetMatrixMap3f& dst_normals,
                                           const ConstVectorSetMatrixMap3f& src_points)
      : b200::ProjectiveICPEntities3f(dst_points, src_points),
        Base(dst_points, dst_normals, src_points, corr_search_, point_corr_weight_eval_, plane_corr_weight_eval_) {}
  SimpleCombinedMetricRigidProjectiveICP3f(const ConstVectorSetMatrixMap3f& dst_points,
                                           const ConstVectorSetMatrixMap3f& dst_normals,
                                           const ConstVectorSetMatrixMap3f& src_points,
                                           const ConstVectorSetMatrixMap3f& src_normals)
      : b200::ProjectiveICPEntities3f(dst_points, src_points),
        Base(dst_points, dst_normals, src_points, src_normals, corr_search_, point_corr_weight_eval_,
             plane_corr_weight_eval_) {}
};

// SimpleCombinedMetricDenseRigidWarpFieldProjectiveICP3f (icp_common_instances.hpp:233-235, :298-299): the dense warp
// field over the projective search of the warped points, with the constructor of its kd-tree sibling
class SimpleCombinedMetricDenseRigidWarpFieldProjectiveICP3f
    : public b200::DenseRigidWarpFieldICP3f<SimpleCombinedMetricDenseRigidWarpFieldProjectiveICP3f,
                                            CorrespondenceSearchProjective<float>> {
public:
  using DenseRigidWarpFieldICP3f::DenseRigidWarpFieldICP3f;
};

// SimpleCombinedMetricSparseRigidWarpFieldProjectiveICP3f (icp_common_instances.hpp:243-245, :327-328): the sparse warp
// field over the projective search of the points warped by the dense field, with the constructor of its kd-tree sibling
class SimpleCombinedMetricSparseRigidWarpFieldProjectiveICP3f
    : public b200::SparseRigidWarpFieldICP3f<SimpleCombinedMetricSparseRigidWarpFieldProjectiveICP3f,
                                             CorrespondenceSearchProjective<float>> {
public:
  using SparseRigidWarpFieldICP3f::SparseRigidWarpFieldICP3f;
};

}  // namespace cilantro
