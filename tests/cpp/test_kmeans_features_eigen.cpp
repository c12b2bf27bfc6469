// VectorSet<float, D> / ConstVectorSetMatrixMap<float, D> for D != 3 (include/cilantro/b200_shims.hpp): layout and
// accessors, and with a real Eigen their conversions from / to Eigen::Matrix<float, D, Dynamic> and MatrixXf. Host only.
#include <cilantro/clustering/kmeans.hpp>

#include <cstdio>
#include <cstdlib>

#define CHECK(c)                                              \
  do {                                                        \
    if (!(c)) {                                               \
      std::fprintf(stderr, "%s:%d: %s\n", __FILE__, __LINE__, #c); \
      std::exit(1);                                           \
    }                                                         \
  } while (0)

int main() {
  cilantro::VectorSet<float, 6> s(6, 4);
  for (size_t c = 0; c < 4; c++)
    for (size_t r = 0; r < 6; r++) s(r, c) = float(10 * c + r);
  CHECK(s.rows() == 6 && s.cols() == 4 && s.data()[6 * 2 + 5] == 25.f);
  cilantro::ConstVectorSetMatrixMap<float, 6> m(s);
  CHECK(m.rows() == 6 && m.cols() == 4 && m.data() == s.data());
  cilantro::VectorSet<float, -1> x(5, 3);
  CHECK(x.rows() == 5 && x.cols() == 3);
  x.resize(7, 2);
  CHECK(x.rows() == 7 && x.cols() == 2);
  cilantro::ConstVectorSetMatrixMap<float, -1> xm(s.data(), 6, 4);
  CHECK(xm.rows() == 6 && xm.cols() == 4);
  cilantro::ConstVectorSetMatrixMap<float, -1> xs(x);
  CHECK(xs.rows() == 7 && xs.cols() == 2);
  static_assert(std::is_same<cilantro::VectorSet<float, 3>, cilantro::VectorSet3f>::value, "3-D stays VectorSet3f");
  static_assert(cilantro::KMeans<float, 6>::Dimension == 6 && cilantro::KMeansXf<>::Dimension == -1, "Dimension");
#ifdef EIGEN_WORLD_VERSION
  Eigen::Matrix<float, 6, Eigen::Dynamic> e = s;  // VectorSet -> Eigen
  CHECK(e.rows() == 6 && e.cols() == 4 && e(5, 2) == 25.f);
  cilantro::VectorSet<float, 6> back(e);  // Eigen -> VectorSet
  CHECK(back(5, 2) == 25.f && back.eigen()(4, 3) == 34.f);
  cilantro::ConstVectorSetMatrixMap<float, 6> em(e);
  CHECK(em.data() == e.data() && em.eigen()(1, 1) == 11.f);
  Eigen::MatrixXf dyn(6, 4);
  dyn = e;
  cilantro::ConstVectorSetMatrixMap<float, Eigen::Dynamic> dm(dyn);
  CHECK(dm.rows() == 6 && dm.cols() == 4 && dm.data() == dyn.data());
  cilantro::VectorSet<float, Eigen::Dynamic> ds(dyn);
  CHECK(ds.rows() == 6 && ds(3, 1) == 13.f);
  Eigen::MatrixXf dback = ds;
  CHECK(dback(2, 3) == 32.f);
  std::printf("eigen adapters (real Eigen) ok\n");
#else
  std::printf("stand-ins ok (Eigen stub: D-dimensional adapters need a real Eigen)\n");
#endif
  return 0;
}
