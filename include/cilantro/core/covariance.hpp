// Same include path as cilantro's core/covariance.hpp: the covariance methods NormalEstimation takes as its
// CovarianceT (core/covariance.hpp:15-371), 3-D float instances. They hold the method's settings; the computation runs
// on the device inside NormalEstimation<float, 3, CovarianceT> (core/normal_estimation.hpp here).
#pragma once
#include <type_traits>

#include "../b200_shims.hpp"

namespace cilantro {

template <typename ScalarT, ptrdiff_t EigenDim>
class Covariance;

// Covariance<float, 3> (:15-182): the plain mean and covariance of a neighbourhood; fewer than
// getMinValidSampleSize() points give NaN.
template <>
class Covariance<float, 3> {
public:
  using Scalar = float;
  enum { Dimension = 3 };
  size_t getMinValidSampleSize() const { return min_sample_size_; }
  Covariance& setMinValidSampleSize(size_t min_size) {
    min_sample_size_ = min_size;
    return *this;
  }

protected:
  size_t min_sample_size_ = 2;
};

template <typename ScalarT, ptrdiff_t EigenDim, typename CovarianceT = Covariance<ScalarT, EigenDim>,
          typename RandomGeneratorT = std::default_random_engine>
class MinimumCovarianceDeterminant;

// MinimumCovarianceDeterminant<float, 3> (:185-371) with the reference's settings and defaults (6 trials,
// 3 refinements, inlier ratio 0.75, no chi-square test). The reference seeds every neighbourhood's generator from
// std::random_device; here setSeed() fixes the seed the per-point generators derive from (DESIGN §4.15), and the
// default seed is drawn from std::random_device once per object.
template <typename CovarianceT, typename RandomGeneratorT>
class MinimumCovarianceDeterminant<float, 3, CovarianceT, RandomGeneratorT> {
public:
  using Scalar = float;
  enum { Dimension = 3 };
  using Covariance = CovarianceT;
  using RandomGenerator = RandomGeneratorT;

  // The whole-set estimate (:210-222, one selection over all the points) is not available on the device; the
  // per-neighbourhood estimate runs inside NormalEstimation.
  template <typename... Args>
  bool operator()(Args&&...) const {
    static_assert(sizeof...(Args) == ~size_t(0), "cilantro_b200: MinimumCovarianceDeterminant is available inside "
                                       "NormalEstimation only; the whole-set operator() is not implemented");
    return false;
  }

  const Covariance& evaluator() const { return compute_mean_and_covariance_; }
  Covariance& evaluator() { return compute_mean_and_covariance_; }
  size_t getMinValidSampleSize() const { return compute_mean_and_covariance_.getMinValidSampleSize(); }
  MinimumCovarianceDeterminant& setMinValidSampleSize(size_t min_size) {
    compute_mean_and_covariance_.setMinValidSampleSize(min_size);
    return *this;
  }
  int getNumberOfTrials() const { return num_trials_; }
  MinimumCovarianceDeterminant& setNumberOfTrials(int num_trials) {
    num_trials_ = num_trials;
    return *this;
  }
  int getNumberOfRefinements() const { return num_refinements_; }
  MinimumCovarianceDeterminant& setNumberOfRefinements(int num_refinements) {
    num_refinements_ = num_refinements;
    return *this;
  }
  float getInlierRatio() const { return inlier_ratio_; }
  MinimumCovarianceDeterminant& setInlierRatio(float inlier_ratio) {
    inlier_ratio_ = inlier_ratio;
    return *this;
  }
  float getChiSquareThreshold() const { return chi_square_threshold_; }
  MinimumCovarianceDeterminant& setChiSquareThreshold(float chi_square_threshold) {
    chi_square_threshold_ = chi_square_threshold;
    return *this;
  }
  // (not in the reference) the seed of the per-point generators
  uint32_t getSeed() const { return seed_; }
  MinimumCovarianceDeterminant& setSeed(uint32_t seed) {
    seed_ = seed;
    return *this;
  }

  cb_mcd_params b200_params() const {
    cb_mcd_params p;
    p.num_trials = num_trials_;
    p.num_refinements = num_refinements_;
    p.inlier_ratio = inlier_ratio_;
    p.chi_square_threshold = chi_square_threshold_;
    p.min_sample_size = (int)std::min<size_t>(getMinValidSampleSize(), 1u << 30);
    p.seed = seed_;
    return p;
  }

protected:
  int num_trials_ = 6;
  int num_refinements_ = 3;
  float inlier_ratio_ = 0.75f;
  float chi_square_threshold_ = -1.0f;
  uint32_t seed_ = b200::random_seed();
  Covariance compute_mean_and_covariance_;
};

}  // namespace cilantro
