// Same include path as cilantro's core/normal_estimation.hpp; the GPU-native drop-in (NormalEstimation3f) lives in
// b200_shims.hpp. NormalEstimation<float, 3, CovarianceT> names it for the plain covariance and adds the robust
// (minimum covariance determinant) instance.
#pragma once
#include "../b200_shims.hpp"
#include "covariance.hpp"

namespace cilantro {

template <typename ScalarT, ptrdiff_t EigenDim, typename CovarianceT = Covariance<ScalarT, EigenDim>,
          typename IndexT = size_t>
class NormalEstimation;

template <typename IndexT>
class NormalEstimation<float, 3, Covariance<float, 3>, IndexT> : public NormalEstimation3f {
public:
  using NormalEstimation3f::NormalEstimation3f;
};

// NormalEstimation<float, 3, MinimumCovarianceDeterminant<float, 3>> (normal_estimation.hpp:11-421) over
// cb_cloud_estimate_normals_mcd: kNN and kNN-in-radius neighbourhoods of at most 128 points. The radius-only
// neighbourhood is not supported on the device: those calls throw.
template <typename CovT, typename RngT, typename IndexT>
class NormalEstimation<float, 3, MinimumCovarianceDeterminant<float, 3, CovT, RngT>, IndexT> {
public:
  using Covariance = MinimumCovarianceDeterminant<float, 3, CovT, RngT>;

  NormalEstimation(const ConstVectorSetMatrixMap3f& points, size_t /*max_leaf_size*/ = 10)
      : n_(points.cols()), points_(points), cloud_(points) {
    const float nan = std::numeric_limits<float>::quiet_NaN();
    view_point_ = Vector3f(nan, nan, nan);
    cov_.setMinValidSampleSize(3);  // :27
  }
  template <typename TreeIndexT>
  explicit NormalEstimation(const KDTree3f<TreeIndexT>& kd_tree) : NormalEstimation(kd_tree.getPointsMatrixMap()) {}

  const Covariance& covarianceMethod() const { return cov_; }
  Covariance& covarianceMethod() { return cov_; }
  const Vector3f& getViewPoint() const { return view_point_; }
  NormalEstimation& setViewPoint(const Vector3f& vp) {
    view_point_ = vp;
    return *this;
  }
  NormalEstimation& setReferenceNormals(const ConstVectorSetMatrixMap3f& ref_normals) {
    if (ref_normals.cols() == n_) {
      ref_normals_.assign(ref_normals.data(), ref_normals.data() + 3 * n_);
      use_ref_ = n_ > 0;
    }
    return *this;
  }

  VectorSet3f getNormalsKNN(size_t k) const { return estimateNormalsKNN(k); }
  VectorSet3f getNormalsRadius(float radius) const { return estimateNormalsRadius(radius); }
  VectorSet3f getNormalsKNNInRadius(size_t k, float radius) const { return estimateNormalsKNNInRadius(k, radius); }

  const NormalEstimation& estimateNormalsAndCurvatureKNN(VectorSet3f& normals, std::vector<float>& curvature,
                                                         size_t k) const {
    return run(&normals, &curvature, k, 0.f);
  }
  const NormalEstimation& estimateNormalsKNN(VectorSet3f& normals, size_t k) const {
    return run(&normals, nullptr, k, 0.f);
  }
  VectorSet3f estimateNormalsKNN(size_t k) const {
    VectorSet3f n;
    run(&n, nullptr, k, 0.f);
    return n;
  }
  const NormalEstimation& estimateCurvatureKNN(std::vector<float>& curvature, size_t k) const {
    return run(nullptr, &curvature, k, 0.f);
  }
  const NormalEstimation& estimateNormalsAndCurvatureRadius(VectorSet3f& normals, std::vector<float>& curvature,
                                                            float radius) const {
    return run(&normals, &curvature, 0, radius);
  }
  const NormalEstimation& estimateNormalsRadius(VectorSet3f& normals, float radius) const {
    return run(&normals, nullptr, 0, radius);
  }
  VectorSet3f estimateNormalsRadius(float radius) const {
    VectorSet3f n;
    run(&n, nullptr, 0, radius);
    return n;
  }
  const NormalEstimation& estimateCurvatureRadius(std::vector<float>& curvature, float radius) const {
    return run(nullptr, &curvature, 0, radius);
  }
  const NormalEstimation& estimateNormalsAndCurvatureKNNInRadius(VectorSet3f& normals, std::vector<float>& curvature,
                                                                 size_t k, float radius) const {
    return run(&normals, &curvature, k, radius);
  }
  const NormalEstimation& estimateNormalsKNNInRadius(VectorSet3f& normals, size_t k, float radius) const {
    return run(&normals, nullptr, k, radius);
  }
  VectorSet3f estimateNormalsKNNInRadius(size_t k, float radius) const {
    VectorSet3f n;
    run(&n, nullptr, k, radius);
    return n;
  }
  const NormalEstimation& estimateCurvatureKNNInRadius(std::vector<float>& curvature, size_t k, float radius) const {
    return run(nullptr, &curvature, k, radius);
  }

private:
  const NormalEstimation& run(VectorSet3f* normals, std::vector<float>* curvature, size_t k, float radius) const {
    if (normals) normals->resize(3, n_);
    if (curvature) curvature->resize(n_);
    if (use_ref_) {  // re-upload the reference normals: the previous call overwrote the cloud's normals
      ConstVectorSetMatrixMap3f ref(ref_normals_);
      cloud_.reset(points_, &ref);
    }
    const cb_mcd_params p = cov_.b200_params();
    b200::check(cb_cloud_estimate_normals_mcd(b200::Context::get(), cloud_.h, (int)std::min<size_t>(k, 1u << 30),
                                              radius, view_point_.data(), use_ref_ ? 1 : 0, &p,
                                              normals ? normals->data() : nullptr,
                                              curvature ? curvature->data() : nullptr, nullptr, nullptr, nullptr),
                "cb_cloud_estimate_normals_mcd");
    return *this;
  }
  size_t n_;
  ConstVectorSetMatrixMap3f points_;
  mutable b200::CloudHandle cloud_;
  Vector3f view_point_;
  std::vector<float> ref_normals_;
  bool use_ref_ = false;
  Covariance cov_;
};

}  // namespace cilantro
