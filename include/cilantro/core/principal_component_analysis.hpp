// Same include path as cilantro's core/principal_component_analysis.hpp. PrincipalComponentAnalysis<float, D>
// (:8-92) for any D, Eigen::Dynamic included, on the device (cb_vectors_pca, cb_vectors_project,
// cb_vectors_reconstruct; DESIGN §4.18). PrincipalComponentAnalysis<float, 3> is the PrincipalComponentAnalysis3f class
// of b200_shims.hpp.
#pragma once
#include <cstring>
#include <type_traits>
#include <vector>

#include "../b200_shims.hpp"
#include "covariance.hpp"

namespace cilantro {

namespace b200 {
template <class T>
struct IsMcd : std::false_type {};
template <typename S, ptrdiff_t D, typename C, typename R>
struct IsMcd<MinimumCovarianceDeterminant<S, D, C, R>> : std::true_type {};

template <long EigenDim>
class PcaD {
public:
  using Scalar = float;
  enum { Dimension = EigenDim };
  using VectorType = DenseF<EigenDim, 1>;
  using CovarianceMatrix = DenseF<EigenDim, EigenDim>;
  using DynamicMatrix = DenseF<kDynamic, kDynamic>;

  template <typename CovarianceT = Covariance<float, EigenDim>>
  PcaD(const ConstVectorSetMatrixMap<float, EigenDim>& data, bool /*parallel*/ = false,
       const CovarianceT& cov_eval = CovarianceT()) {
    static_assert(!IsMcd<CovarianceT>::value, "cilantro_b200: PrincipalComponentAnalysis with a "
                                              "MinimumCovarianceDeterminant cov_eval is not implemented");
    compute(data, nullptr, cov_eval.getMinValidSampleSize());
  }
  template <typename ContainerT, typename CovarianceT = Covariance<float, EigenDim>,
            typename = decltype(std::declval<const ContainerT&>().begin())>
  PcaD(const ConstVectorSetMatrixMap<float, EigenDim>& data, const ContainerT& subset, bool /*parallel*/ = false,
       const CovarianceT& cov_eval = CovarianceT()) {
    static_assert(!IsMcd<CovarianceT>::value, "cilantro_b200: PrincipalComponentAnalysis with a "
                                              "MinimumCovarianceDeterminant cov_eval is not implemented");
    std::vector<uint64_t> idx;
    for (auto it = subset.begin(); it != subset.end(); ++it) idx.push_back((uint64_t)*it);
    compute(data, &idx, cov_eval.getMinValidSampleSize());
  }

  const VectorType& getDataMean() const { return mean_; }
  const CovarianceMatrix& getDataCovariance() const { return cov_; }
  const VectorType& getEigenValues() const { return evals_; }
  const CovarianceMatrix& getEigenVectors() const { return evecs_; }

  // project(points, target_dim) (:46-50): target_dim x N, of any D x N float set (data(), rows(), cols())
  template <typename PointsT>
  DynamicMatrix project(const PointsT& points, size_t target_dim) const {
    DynamicMatrix out;
    out.resize(target_dim, points.cols());
    map(points.data(), points.rows(), points.cols(), (int)target_dim, true, out.data());
    return out;
  }
  // project<DimOut>(points) (:52-57)
  template <long EigenDimOut>
  typename std::enable_if<EigenDimOut != kDynamic, VectorSet<float, EigenDimOut>>::type project(
      const ConstVectorSetMatrixMap<float, EigenDim>& points) const {
    VectorSet<float, EigenDimOut> out(EigenDimOut, points.cols());
    map(points.data(), points.rows(), points.cols(), (int)EigenDimOut, true, out.data());
    return out;
  }
  // reconstruct(points) (:59-62): D x N from the first points.rows() components, of any k x N float set
  template <typename PointsT>
  DynamicMatrix reconstruct(const PointsT& points) const {
    DynamicMatrix out;
    out.resize(dim_, points.cols());
    map(points.data(), points.rows(), points.cols(), (int)dim_, false, out.data());
    return out;
  }
  // reconstruct<DimIn>(points) (:64-68)
  template <long EigenDimIn>
  typename std::enable_if<EigenDimIn != kDynamic, VectorSet<float, EigenDim>>::type reconstruct(
      const ConstVectorSetMatrixMap<float, EigenDimIn>& points) const {
    VectorSet<float, EigenDim> out(dim_, points.cols());
    map(points.data(), points.rows(), points.cols(), (int)dim_, false, out.data());
    return out;
  }

private:
  void compute(const ConstVectorSetMatrixMap<float, EigenDim>& data, const std::vector<uint64_t>* subset,
               size_t min_size) {
    dim_ = data.rows();
    const size_t D = dim_;
    VectorsHandle v(data.data(), data.cols(), D);
    mean_.resize(D, 1);
    cov_.resize(D, D);
    evals_.resize(D, 1);
    evecs_.resize(D, D);
    evecs_rm_.resize(D * D);
    const uint64_t none = 0;  // a non-null pointer for an empty subset
    const uint64_t* sp = subset ? (subset->empty() ? &none : subset->data()) : nullptr;
    check(cb_vectors_pca(Context::get(), v.h, sp, subset ? subset->size() : 0, min_size, mean_.data(), cov_.data(),
                         evals_.data(), evecs_rm_.data()),
          "cb_vectors_pca");
    for (size_t i = 0; i < D; i++)
      for (size_t j = 0; j < D; j++) evecs_(i, j) = evecs_rm_[i * D + j];  // row-major -> column-major
  }
  // points (rows x n, column-major = n x rows row-major) through the basis into out (n x dout row-major)
  void map(const float* points, size_t rows, size_t n, int k, bool project, float* out) const {
    VectorsHandle x(points, n, rows);
    if (project)
      check(cb_vectors_project(Context::get(), x.h, mean_.data(), evecs_rm_.data(), k, out, nullptr),
            "cb_vectors_project");
    else
      check(cb_vectors_reconstruct(Context::get(), x.h, mean_.data(), evecs_rm_.data(), k, out, nullptr),
            "cb_vectors_reconstruct");
  }

  size_t dim_ = 0;
  VectorType mean_, evals_;
  CovarianceMatrix cov_, evecs_;
  std::vector<float> evecs_rm_;  // the C ABI's row-major copy of the eigenvectors
};

template <class ScalarT, long EigenDim>
struct PcaInstance {
  static_assert(std::is_same<ScalarT, float>::value, "cilantro_b200 provides float PrincipalComponentAnalysis only "
                                                     "(no double instances)");
  using type = PcaD<EigenDim>;
};
template <>
struct PcaInstance<float, 3> {
  using type = PrincipalComponentAnalysis3f;
};
}  // namespace b200

template <typename ScalarT, long EigenDim>
using PrincipalComponentAnalysis = typename b200::PcaInstance<ScalarT, EigenDim>::type;
using PrincipalComponentAnalysis2f = PrincipalComponentAnalysis<float, 2>;
using PrincipalComponentAnalysisXf = PrincipalComponentAnalysis<float, b200::kDynamic>;

}  // namespace cilantro
