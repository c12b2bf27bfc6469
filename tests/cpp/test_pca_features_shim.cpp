// The C++ drop-ins of covariance and PCA over D-dimensional rows (Covariance<float, D>, PrincipalComponentAnalysis<float,
// D>, PrincipalComponentAnalysis2f / Xf), run on the device; tests/test_pca_features_shims.py compares the output with
// the C ABI through capi bit for bit.
//
//   test_pca_features_shim in.bin out.bin
//   in:  int64 n, D, k, m; float32 rows [n x D] (row-major = the D x n column-major set); int64 subset [m]
//   out: float32, for the whole set and then the subset: mean [D], cov [D x D], eigenvalues [D], eigenvectors
//        [D x D] (all column-major); then Covariance::operator() mean and cov of the whole set; then the projection
//        [k x n] and the reconstruction of that projection [D x n]
#include <cilantro/core/covariance.hpp>
#include <cilantro/core/principal_component_analysis.hpp>

#include <cstdint>
#include <cstdio>
#include <type_traits>
#include <vector>

static_assert(std::is_same<cilantro::PrincipalComponentAnalysis<float, 3>, cilantro::PrincipalComponentAnalysis3f>::value,
              "PrincipalComponentAnalysis<float, 3> is PrincipalComponentAnalysis3f");

template <class M>
static void put(FILE* o, const M& m) {
  std::fwrite(m.data(), sizeof(float), m.rows() * m.cols(), o);
}

template <long D>
static int run(const std::vector<float>& rows, size_t n, size_t dim, size_t k, const std::vector<size_t>& subset,
               FILE* o) {
  const cilantro::ConstVectorSetMatrixMap<float, D> data(rows.data(), dim, n);
  cilantro::Covariance<float, D> cov_eval;
  cov_eval.setMinValidSampleSize(2);
  const cilantro::PrincipalComponentAnalysis<float, D> whole(data, false, cov_eval);
  const cilantro::PrincipalComponentAnalysis<float, D> part(data, subset);
  for (const auto* p : {&whole, &part}) {
    put(o, p->getDataMean());
    put(o, p->getDataCovariance());
    put(o, p->getEigenValues());
    put(o, p->getEigenVectors());
  }
  typename cilantro::Covariance<float, D>::VectorType mean;
  typename cilantro::Covariance<float, D>::MatrixType cov;
  if (!cov_eval(data, mean, cov)) return 1;
  put(o, mean);
  put(o, cov);
  const auto proj = whole.project(data, k);
  put(o, proj);
  put(o, whole.reconstruct(proj));
  // the iterator overload gives the container overload's bits
  typename cilantro::Covariance<float, D>::VectorType m2;
  typename cilantro::Covariance<float, D>::MatrixType c2;
  cov_eval(data, subset.begin(), subset.end(), m2, c2);
  for (size_t i = 0; i < dim; i++)
    if (!(m2.data()[i] == part.getDataMean().data()[i] || m2.data()[i] != m2.data()[i])) return 2;
  return 0;
}

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  int64_t hdr[4];
  if (std::fread(hdr, sizeof(int64_t), 4, f) != 4) return 2;
  const size_t n = (size_t)hdr[0], D = (size_t)hdr[1], k = (size_t)hdr[2], m = (size_t)hdr[3];
  std::vector<float> rows(n * D);
  std::vector<int64_t> sub64(m);
  if (std::fread(rows.data(), sizeof(float), rows.size(), f) != rows.size()) return 2;
  if (std::fread(sub64.data(), sizeof(int64_t), m, f) != m) return 2;
  std::fclose(f);
  const std::vector<size_t> subset(sub64.begin(), sub64.end());
  FILE* o = std::fopen(argv[2], "wb");
  if (!o) return 2;
  int rc;
  if (D == 2) {
    static_assert(std::is_same<cilantro::PrincipalComponentAnalysis2f, cilantro::PrincipalComponentAnalysis<float, 2>>::value, "");
    rc = run<2>(rows, n, D, k, subset, o);
  } else if (D == 6) {
    rc = run<6>(rows, n, D, k, subset, o);
  } else {
    rc = run<cilantro::b200::kDynamic>(rows, n, D, k, subset, o);
  }
  std::fclose(o);
  if (rc != 0) return rc;
  if (D == 3) {  // PrincipalComponentAnalysisXf on 3 rows equals PrincipalComponentAnalysis3f bit for bit
    const cilantro::PrincipalComponentAnalysisXf x(cilantro::ConstVectorSetMatrixMap<float, cilantro::b200::kDynamic>(rows.data(), 3, n));
    const cilantro::PrincipalComponentAnalysis3f p3(cilantro::ConstVectorSetMatrixMap3f(rows.data(), n));
    for (int i = 0; i < 3; i++) {
      if (x.getDataMean().data()[i] != p3.getDataMean()[i] || x.getEigenValues().data()[i] != p3.getEigenValues()[i]) return 3;
      for (int j = 0; j < 3; j++)
        if (x.getDataCovariance()(i, j) != p3.getDataCovariance()[3 * i + j] ||
            x.getEigenVectors()(i, j) != p3.getEigenVectors()[3 * i + j])
          return 3;
    }
    std::printf("PrincipalComponentAnalysisXf on 3 rows = PrincipalComponentAnalysis3f\n");
  }
  std::printf("pca features shim: n = %zu, D = %zu, k = %zu, subset %zu\n", n, D, k, m);
  return 0;
}
