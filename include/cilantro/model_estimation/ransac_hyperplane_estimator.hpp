// Same include path as cilantro's model_estimation/ransac_hyperplane_estimator.hpp: HyperplaneRANSACEstimator3f<> /
// PlaneRANSACEstimator3f<> on the device (cb_ransac_plane, DESIGN §4.12).
#pragma once
#include <cmath>
#include <limits>
#include <vector>

#include "../b200_shims.hpp"

namespace cilantro {

// Stand-in for Eigen::Hyperplane<float, 3>: normal . p + offset = 0, coefficients (n0, n1, n2, d).
class Hyperplane3f {
public:
  Hyperplane3f() { c_.fill(std::numeric_limits<float>::quiet_NaN()); }
  explicit Hyperplane3f(const float* coeffs4) { std::memcpy(c_.data(), coeffs4, sizeof(float) * 4); }
  Hyperplane3f(const Vector3f& n, float d) : c_{n[0], n[1], n[2], d} {}
  Vector3f normal() const { return Vector3f(c_[0], c_[1], c_[2]); }
  float offset() const { return c_[3]; }
  float& offset() { return c_[3]; }
  const std::array<float, 4>& coeffs() const { return c_; }
  std::array<float, 4>& coeffs() { return c_; }
  // the residual convention of cb_plane_residuals: ((n0 x) + ((n1 y) + (n2 z))) + d
  float signedDistance(const Vector3f& p) const { return (c_[0] * p[0] + (c_[1] * p[1] + c_[2] * p[2])) + c_[3]; }
  float absDistance(const Vector3f& p) const { return std::fabs(signedDistance(p)); }
#ifdef CILANTRO_B200_HAS_EIGEN
  Hyperplane3f(const Eigen::Hyperplane<float, 3>& h) {
    for (int i = 0; i < 4; i++) c_[i] = h.coeffs()(i);
  }
  operator Eigen::Hyperplane<float, 3>() const {
    Eigen::Hyperplane<float, 3> h;
    for (int i = 0; i < 4; i++) h.coeffs()(i) = c_[i];
    return h;
  }
#endif

private:
  std::array<float, 4> c_;
};

// HyperplaneRANSACEstimator<float, 3, IndexT> (ransac_hyperplane_estimator.hpp:9-112) with the surface of
// RandomSampleConsensusBase (b200::RansacEstimator): threshold 0.1; setSampleSize is not offered.
template <typename IndexT = size_t>
class HyperplaneRANSACEstimator3f
    : public b200::RansacEstimator<HyperplaneRANSACEstimator3f<IndexT>, Hyperplane3f, IndexT> {
  using Base = b200::RansacEstimator<HyperplaneRANSACEstimator3f<IndexT>, Hyperplane3f, IndexT>;
  friend Base;

public:
  using typename Base::IndexVector;
  using typename Base::ResidualVector;

  HyperplaneRANSACEstimator3f(const ConstVectorSetMatrixMap3f& points)
      : Base(points.cols(), 0.1f), points_(points), cloud_(points) {}

  // estimateModel (:21-42): the PCA plane of all points / of the listed points
  HyperplaneRANSACEstimator3f& estimateModel(Hyperplane3f& model) {
    model = pca_plane(PrincipalComponentAnalysis3f(points_));
    return *this;
  }
  Hyperplane3f estimateModel() { return pca_plane(PrincipalComponentAnalysis3f(points_)); }
  HyperplaneRANSACEstimator3f& estimateModel(const IndexVector& sample_ind, Hyperplane3f& model) {
    model = pca_plane(PrincipalComponentAnalysis3f(points_, sample_ind));
    return *this;
  }
  Hyperplane3f estimateModel(const IndexVector& sample_ind) {
    return pca_plane(PrincipalComponentAnalysis3f(points_, sample_ind));
  }
  // computeResiduals (:44-62)
  HyperplaneRANSACEstimator3f& computeResiduals(const Hyperplane3f& model, ResidualVector& residuals) {
    residuals.resize(this->n_);
    b200::check(cb_plane_residuals(b200::Context::get(), cloud_.h, model.coeffs().data(), this->thresh_,
                                   residuals.data(), nullptr, nullptr),
                "cb_plane_residuals");
    return *this;
  }
  ResidualVector computeResiduals(const Hyperplane3f& model) {
    ResidualVector r;
    computeResiduals(model, r);
    return r;
  }
  size_t getDataPointsCount() const { return this->n_; }

private:
  size_t run(uint64_t* inliers, float* residuals) {
    cb_ransac_plane_result r;
    b200::check(cb_ransac_plane(b200::Context::get(), cloud_.h, this->seed_, this->target_, this->max_iter_,
                                this->thresh_, this->re_estimate_ ? 1 : 0, &r, inliers, residuals),
                "cb_ransac_plane");
    this->model_ = Hyperplane3f(r.plane);
    this->iterations_ = r.iterations;
    return r.num_inliers;
  }
  // estimate_params_ (:96-110): normal = the last eigenvector column, offset = -(normal . mean)
  static Hyperplane3f pca_plane(const PrincipalComponentAnalysis3f& pca) {
    const auto& V = pca.getEigenVectors();
    const Vector3f n(V[2], V[5], V[8]), m = pca.getDataMean();
    return Hyperplane3f(n, -(n[0] * m[0] + (n[1] * m[1] + n[2] * m[2])));
  }
  ConstVectorSetMatrixMap3f points_;
  b200::CloudHandle cloud_;
};

template <typename IndexT = size_t>
using PlaneRANSACEstimator3f = HyperplaneRANSACEstimator3f<IndexT>;

}  // namespace cilantro
