// The robust normal-estimation shim (include/cilantro/core/normal_estimation.hpp with core/covariance.hpp) in the
// reference example's call sequence (examples/robust_normal_estimation.cpp), and PointCloud3f::removeInvalidNormals.
// tests/test_robust_normals_shims.py builds and runs it.
//
//   test_robust_normals_shim <points.bin> <seed>
// points.bin: packed float32 xyz. Prints "normals <bit patterns...>" and "kept <count>".
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <cilantro/core/covariance.hpp>
#include <cilantro/core/normal_estimation.hpp>
#include <cilantro/utilities/point_cloud.hpp>

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  std::FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<float> xyz;
  float buf[3];
  while (std::fread(buf, sizeof(float), 3, f) == 3) xyz.insert(xyz.end(), buf, buf + 3);
  std::fclose(f);
  cilantro::PointCloud3f cloud;
  cloud.points = cilantro::VectorSet3f(3, xyz.size() / 3);
  std::memcpy(cloud.points.data(), xyz.data(), xyz.size() * sizeof(float));

  cilantro::KDTree3f<> tree(cloud.points);
  cilantro::NormalEstimation<float, 3, cilantro::MinimumCovarianceDeterminant<float, 3>> ne(tree);
  ne.setViewPoint(cilantro::Vector3f(0.f, 0.f, 0.f));
  ne.covarianceMethod().setChiSquareThreshold(6.25).setNumberOfTrials(2).setNumberOfRefinements(1);
  ne.covarianceMethod().setSeed((uint32_t)std::strtoul(argv[2], nullptr, 10));
  if (ne.covarianceMethod().getMinValidSampleSize() != 3 || ne.covarianceMethod().getNumberOfTrials() != 2 ||
      ne.covarianceMethod().getNumberOfRefinements() != 1 || ne.covarianceMethod().getInlierRatio() != 0.75f ||
      ne.covarianceMethod().getChiSquareThreshold() != 6.25f) {
    std::printf("FAIL: settings\n");
    return 1;
  }
  cloud.normals = ne.getNormalsKNN(12);
  std::printf("normals %zu", cloud.normals.cols());
  for (size_t i = 0; i < 3 * cloud.normals.cols(); i++) {
    uint32_t u;
    std::memcpy(&u, cloud.normals.data() + i, 4);
    std::printf(" %u", u);
  }
  std::printf("\n");
  // the plain instance is the existing NormalEstimation3f under the reference's template name
  cilantro::NormalEstimation<float, 3> plain(cloud.points);
  if (plain.getNormalsKNN(12).cols() != cloud.size()) return 1;
  // radius-only neighbourhoods are not supported by the robust instance
  bool threw = false;
  try {
    ne.getNormalsRadius(0.01f);
  } catch (const std::runtime_error&) {
    threw = true;
  }
  if (!threw) {
    std::printf("FAIL: radius-only call did not throw\n");
    return 1;
  }
  cloud.removeInvalidNormals();
  std::printf("kept %zu\n", cloud.size());
  return 0;
}
