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
// RandomSampleConsensusBase (ransac_base.hpp:10-187). Sample size 3 (setSampleSize is not offered); the seed of the
// sampler is injected with setRandomSeed (the reference draws it from std::random_device).
template <typename IndexT = size_t>
class HyperplaneRANSACEstimator3f {
public:
  using Model = Hyperplane3f;
  using ResidualScalar = float;
  using ResidualVector = std::vector<float>;
  using Index = IndexT;
  using IndexVector = std::vector<IndexT>;

  HyperplaneRANSACEstimator3f(const ConstVectorSetMatrixMap3f& points)
      : n_(points.cols()), points_(points), cloud_(points), target_(n_ / 2 + n_ % 2), seed_(b200::random_seed()) {}

  size_t getSampleSize() const { return 3; }
  size_t getTargetInlierCount() const { return target_; }
  HyperplaneRANSACEstimator3f& setTargetInlierCount(size_t c) { target_ = c; return *this; }
  size_t getMaxNumberOfIterations() const { return max_iter_; }
  HyperplaneRANSACEstimator3f& setMaxNumberOfIterations(size_t m) { max_iter_ = m; return *this; }
  float getMaxInlierResidual() const { return thresh_; }
  HyperplaneRANSACEstimator3f& setMaxInlierResidual(float t) { thresh_ = t; return *this; }
  bool getReEstimationStep() const { return re_estimate_; }
  HyperplaneRANSACEstimator3f& setReEstimationStep(bool b) { re_estimate_ = b; return *this; }
  HyperplaneRANSACEstimator3f& setRandomSeed(uint32_t s) { seed_ = s; return *this; }

  HyperplaneRANSACEstimator3f& estimate() {
    if (target_ > n_) target_ = n_;  // ransac_base.hpp:68
    cb_ransac_plane_result r;
    std::vector<uint64_t> inl(n_);
    residuals_.resize(n_);
    b200::check(cb_ransac_plane(b200::Context::get(), cloud_.h, seed_, target_, max_iter_, thresh_, re_estimate_ ? 1 : 0,
                                &r, inl.data(), residuals_.data()),
                "cb_ransac_plane");
    model_ = Hyperplane3f(r.plane);
    iterations_ = r.iterations;
    inliers_.assign(inl.begin(), inl.begin() + r.num_inliers);
    return *this;
  }
  HyperplaneRANSACEstimator3f& estimate(float max_residual, size_t target_inlier_count, size_t max_iter) {  // :133-140
    thresh_ = max_residual;
    target_ = target_inlier_count;
    max_iter_ = max_iter;
    return estimate();
  }

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
    residuals.resize(n_);
    b200::check(cb_plane_residuals(b200::Context::get(), cloud_.h, model.coeffs().data(), thresh_, residuals.data(),
                                   nullptr, nullptr),
                "cb_plane_residuals");
    return *this;
  }
  ResidualVector computeResiduals(const Hyperplane3f& model) {
    ResidualVector r;
    computeResiduals(model, r);
    return r;
  }
  size_t getDataPointsCount() const { return n_; }

  const HyperplaneRANSACEstimator3f& getEstimationResults(Model& model, ResidualVector& residuals,
                                                          IndexVector& inliers) const {
    model = model_;
    residuals = residuals_;
    inliers = inliers_;
    return *this;
  }
  const Model& getModel() const { return model_; }
  const HyperplaneRANSACEstimator3f& getModel(Model& m) const { m = model_; return *this; }
  const ResidualVector& getModelResiduals() const { return residuals_; }
  const HyperplaneRANSACEstimator3f& getModelResiduals(ResidualVector& r) const { r = residuals_; return *this; }
  const IndexVector& getModelInliers() const { return inliers_; }
  const HyperplaneRANSACEstimator3f& getModelInliers(IndexVector& i) const { i = inliers_; return *this; }
  bool targetInlierCountAchieved() const { return inliers_.size() >= target_; }
  size_t getNumberOfPerformedIterations() const { return iterations_; }
  size_t getNumberOfInliers() const { return inliers_.size(); }

private:
  // estimate_params_ (:96-110): normal = the last eigenvector column, offset = -(normal . mean)
  static Hyperplane3f pca_plane(const PrincipalComponentAnalysis3f& pca) {
    const auto& V = pca.getEigenVectors();
    const Vector3f n(V[2], V[5], V[8]), m = pca.getDataMean();
    return Hyperplane3f(n, -(n[0] * m[0] + (n[1] * m[1] + n[2] * m[2])));
  }
  size_t n_;
  ConstVectorSetMatrixMap3f points_;
  b200::CloudHandle cloud_;
  size_t target_, max_iter_ = 100, iterations_ = 0;  // ransac_hyperplane_estimator.hpp:18
  float thresh_ = 0.1f;
  bool re_estimate_ = true;
  uint32_t seed_;
  Model model_;
  ResidualVector residuals_;
  IndexVector inliers_;
};

template <typename IndexT = size_t>
using PlaneRANSACEstimator3f = HyperplaneRANSACEstimator3f<IndexT>;

}  // namespace cilantro
