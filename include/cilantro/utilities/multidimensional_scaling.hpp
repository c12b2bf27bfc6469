// Same include path as cilantro's utilities/multidimensional_scaling.hpp. Classical multidimensional scaling on the
// device (cb_vectors_mds; DESIGN §4.19): estimateEmbeddingDimensionEigengap (:9-31),
// computeDistancePreservingSpectralEmbedding (:35-83) and MultidimensionalScaling<float, D> (:86-121) with the
// SpectralEmbeddingBase getters (core/spectral_embedding_base.hpp:9-26), for D = 2, 3, ... and Eigen::Dynamic.
#pragma once
#include <algorithm>
#include <cstring>
#include <limits>
#include <stdexcept>
#include <type_traits>
#include <vector>

#include "../b200_shims.hpp"

namespace cilantro {

// The dimension whose following eigenvalue gap is the largest, or max_dim when the values spread less than epsilon.
// eigenvalues: any vector with rows() and operator[].
template <class VectorT>
size_t estimateEmbeddingDimensionEigengap(const VectorT& eigenvalues, size_t max_dim) {
  using S = typename std::decay<decltype(eigenvalues[0])>::type;
  const size_t m = (size_t)eigenvalues.rows();
  S lo = std::numeric_limits<S>::infinity(), hi = -std::numeric_limits<S>::infinity();
  S best = -std::numeric_limits<S>::infinity();
  size_t ind = 0;
  for (size_t i = 0; i + 1 < m; i++) {
    const S gap = eigenvalues[i] - eigenvalues[i + 1];
    if (gap > best) {
      best = gap;
      ind = i;
    }
    lo = std::min(lo, (S)eigenvalues[i]);
    hi = std::max(hi, (S)eigenvalues[i]);
  }
  if (eigenvalues[m - 1] < lo) lo = eigenvalues[m - 1];
  if (eigenvalues[m - 1] > hi) hi = eigenvalues[m - 1];
  if (hi - lo < std::numeric_limits<S>::epsilon()) return max_dim;
  return ind + 1;
}

namespace b200 {
template <class ScalarT>
struct MdsFloat {
  static_assert(std::is_same<ScalarT, float>::value,
                "cilantro_b200 provides float MultidimensionalScaling only (no double instances)");
};

// distances: any column-major float n x n matrix (data(), rows(), cols()). embedded (dim x n) and eigenvalues (nev)
// are resized and filled. nev outside [1, n - 1] throws std::invalid_argument, as the reference's eigen-solver does.
template <class MatrixT, class SetT, class VecT>
void mds(const MatrixT& distances, size_t max_dim, bool estimate_dim, bool distances_are_squared, SetT& embedded,
         VecT& eigenvalues) {
  const size_t n = (size_t)distances.rows();
  if ((size_t)distances.cols() != n) throw std::invalid_argument("MultidimensionalScaling: distances must be square");
  const size_t nev = estimate_dim ? std::min(max_dim + 1, n - 1) : max_dim;
  if (n < 2 || nev < 1 || nev > n - 1 || (estimate_dim && max_dim > n - 1))
    throw std::invalid_argument("MultidimensionalScaling: number of eigenvalues out of [1, n - 1]");
  // the C ABI takes rows: the transpose of the column-major input
  std::vector<float> rows(n * n);
  const float* src = distances.data();
  constexpr size_t kB = 64;
  for (size_t j0 = 0; j0 < n; j0 += kB)
    for (size_t i0 = 0; i0 < n; i0 += kB)
      for (size_t j = j0; j < std::min(n, j0 + kB); j++)
        for (size_t i = i0; i < std::min(n, i0 + kB); i++) rows[i * n + j] = src[j * n + i];
  VectorsHandle v(rows.data(), n, n);
  std::vector<float>().swap(rows);
  std::vector<float> ev(nev), emb(n * std::max<size_t>(max_dim, 1));
  size_t got_nev = 0, dim = 0;
  check(cb_vectors_mds(Context::get(), v.h, max_dim, estimate_dim ? 1 : 0, distances_are_squared ? 1 : 0, ev.data(),
                       &got_nev, &dim, emb.data(), nullptr),
        "cb_vectors_mds");
  eigenvalues.resize(got_nev, 1);
  for (size_t i = 0; i < got_nev; i++) eigenvalues.data()[i] = ev[i];
  embedded.resize(dim, n);  // dim x n column-major: the n x dim rows of the C ABI
  if (n * dim != 0) std::memcpy(embedded.data(), emb.data(), n * dim * sizeof(float));
}
}  // namespace b200

// computeDistancePreservingSpectralEmbedding (:35-83)
template <typename ScalarT, long EigenDim = b200::kDynamic, class MatrixT, class SetT, class VecT>
void computeDistancePreservingSpectralEmbedding(const MatrixT& distances, size_t max_dim, bool estimate_dim,
                                                bool distances_are_squared, SetT& embedded_points,
                                                VecT& computed_eigenvalues) {
  (void)sizeof(b200::MdsFloat<ScalarT>);
  b200::mds(distances, max_dim, estimate_dim, distances_are_squared, embedded_points, computed_eigenvalues);
}

template <typename ScalarT, long EigenDim = b200::kDynamic>
class MultidimensionalScaling {
  static_assert(std::is_same<ScalarT, float>::value,
                "cilantro_b200 provides float MultidimensionalScaling only (no double instances)");

public:
  using Scalar = ScalarT;
  enum { Dimension = EigenDim };
  using EmbeddedSet = VectorSet<float, EigenDim>;
  // a column vector with data(), rows(), operator[] and operator() (the reference's Vector<float, EigenDim>)
  using EigenValues = b200::DenseMatrixF<EigenDim, 1>;

  // fixed embedding dimension EigenDim (:93-100)
  template <class MatrixT, long Dim = EigenDim, class = typename std::enable_if<Dim != b200::kDynamic>::type>
  MultidimensionalScaling(const MatrixT& distances, bool distances_are_squared = true) {
    b200::mds(distances, (size_t)EigenDim, false, distances_are_squared, embedded_points_, computed_eigenvalues_);
  }

  // run-time dimension (:105-118): max_dim in [1, n - 1], else dimension 2 without estimation
  template <class MatrixT, long Dim = EigenDim, class = typename std::enable_if<Dim == b200::kDynamic>::type>
  MultidimensionalScaling(const MatrixT& distances, size_t max_dim, bool estimate_dim = false,
                          bool distances_are_squared = true) {
    if (max_dim > 0 && max_dim < (size_t)distances.rows())
      b200::mds(distances, max_dim, estimate_dim, distances_are_squared, embedded_points_, computed_eigenvalues_);
    else
      b200::mds(distances, 2, false, distances_are_squared, embedded_points_, computed_eigenvalues_);
  }

  const EmbeddedSet& getEmbeddedPoints() const { return embedded_points_; }
  const EigenValues& getComputedEigenValues() const { return computed_eigenvalues_; }
  size_t getEmbeddingDimension() const { return (size_t)embedded_points_.rows(); }

private:
  EmbeddedSet embedded_points_;
  EigenValues computed_eigenvalues_;
};

using MultidimensionalScaling2f = MultidimensionalScaling<float, 2>;
using MultidimensionalScaling3f = MultidimensionalScaling<float, 3>;
using MultidimensionalScalingXf = MultidimensionalScaling<float, b200::kDynamic>;
// the double aliases name the class; using one is the compile-time error above
using MultidimensionalScaling2d = MultidimensionalScaling<double, 2>;
using MultidimensionalScaling3d = MultidimensionalScaling<double, 3>;
using MultidimensionalScalingXd = MultidimensionalScaling<double, b200::kDynamic>;

}  // namespace cilantro
