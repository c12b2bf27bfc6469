// Same include path as cilantro's core/covariance.hpp: the covariance methods NormalEstimation takes as its
// CovarianceT (core/covariance.hpp:15-371), 3-D float instances. They hold the method's settings; the computation runs
// on the device inside NormalEstimation<float, 3, CovarianceT> (core/normal_estimation.hpp here).
#pragma once
#include <cstdint>
#include <iterator>
#include <type_traits>
#include <vector>

#include "../b200_shims.hpp"

namespace cilantro {

template <typename ScalarT, ptrdiff_t EigenDim>
class Covariance;

// Covariance<float, D> (:15-182) for any D, Eigen::Dynamic included: the mean and (n - 1)-normalised covariance of a
// vector set, whole or the listed columns, on the device (cb_vectors_mean_cov, DESIGN §4.18; at D = 3 the bits of
// cb_mean_cov). Fewer than getMinValidSampleSize() points give NaN and false. NormalEstimation<float, 3, ...> takes
// Covariance<float, 3> as the holder of that setting and runs its own per-neighbourhood kernel.
template <ptrdiff_t EigenDim>
class Covariance<float, EigenDim> {
public:
  using Scalar = float;
  enum { Dimension = EigenDim };
  using VectorType = b200::DenseF<EigenDim, 1>;
  using MatrixType = b200::DenseF<EigenDim, EigenDim>;

  size_t getMinValidSampleSize() const { return min_sample_size_; }
  Covariance& setMinValidSampleSize(size_t min_size) {
    min_sample_size_ = min_size;
    return *this;
  }

  // whole set (:30-80)
  bool operator()(const ConstVectorSetMatrixMap<float, EigenDim>& points, VectorType& mean, MatrixType& cov,
                  bool /*parallel*/ = false) const {
    return run(points, nullptr, mean, cov);
  }
  // the columns [begin, end) lists (:83-172); duplicates count twice
  template <typename IteratorT, typename = typename std::iterator_traits<IteratorT>::iterator_category>
  bool operator()(const ConstVectorSetMatrixMap<float, EigenDim>& points, IteratorT begin, IteratorT end,
                  VectorType& mean, MatrixType& cov, bool /*parallel*/ = false) const {
    std::vector<uint64_t> idx;
    for (IteratorT it = begin; it != end; ++it) idx.push_back((uint64_t)*it);
    return run(points, &idx, mean, cov);
  }
  // a container of column indices (:174-179)
  template <typename ContainerT, typename = decltype(std::declval<const ContainerT&>().begin())>
  bool operator()(const ConstVectorSetMatrixMap<float, EigenDim>& points, const ContainerT& subset, VectorType& mean,
                  MatrixType& cov, bool parallel = false) const {
    return (*this)(points, subset.begin(), subset.end(), mean, cov, parallel);
  }

protected:
  // subset nullptr: the whole set
  bool run(const ConstVectorSetMatrixMap<float, EigenDim>& points, const std::vector<uint64_t>* subset,
           VectorType& mean, MatrixType& cov) const {
    const size_t D = points.rows();
    b200::VectorsHandle v(points.data(), points.cols(), D);
    mean.resize(D, 1);
    cov.resize(D, D);
    const uint64_t none = 0;  // a non-null pointer for an empty subset
    const uint64_t* sp = subset ? (subset->empty() ? &none : subset->data()) : nullptr;
    const int rc = cb_vectors_mean_cov(b200::Context::get(), v.h, sp, subset ? subset->size() : 0, min_sample_size_,
                                       mean.data(), cov.data());  // cov is symmetric: either storage order
    b200::check(rc, "cb_vectors_mean_cov");
    return rc == 1;
  }
  size_t min_sample_size_ = 2;
};

template <ptrdiff_t EigenDim>
class Covariance<double, EigenDim> {
  static_assert(EigenDim != EigenDim, "cilantro_b200 provides float Covariance only (no double instances)");
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
