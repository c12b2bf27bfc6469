// Robust normal estimation through the shims, the recipe of the reference's examples/robust_normal_estimation.cpp:
// PLY (or a synthetic plane with off-plane outliers) -> gridDownsample(0.005) -> NormalEstimation with
// MinimumCovarianceDeterminant (k = 12, view point at the origin, chi-square 6.25, 2 trials, 1 refinement)
// -> removeInvalidNormals().
//   make -C examples robust_normal_estimation_cloud && ./examples/robust_normal_estimation_cloud [cloud.ply]
#include <cstdio>
#include <random>

#include <cilantro/utilities/point_cloud.hpp>
#include <cilantro/utilities/timer.hpp>

int main(int argc, char** argv) {
  cilantro::PointCloud3f cloud;
  if (argc > 1) {
    cloud = cilantro::PointCloud3f(argv[1]);
  } else {  // a plane z = 1 seen from the origin, 20 % of the points pushed off it by 1-3 cm
    std::mt19937 rng(1);
    std::uniform_real_distribution<float> u(-0.5f, 0.5f), off(0.01f, 0.03f);
    std::normal_distribution<float> noise(0.f, 0.0003f);
    const size_t n = 200000;
    cloud.points.resize(3, n);
    for (size_t i = 0; i < n; i++)
      cloud.points.setCol(i, cilantro::Vector3f(u(rng), u(rng), 1.f + noise(rng) + (i % 5 == 0 ? off(rng) : 0.f)));
  }
  if (cloud.isEmpty()) {
    std::printf("Input cloud is empty!\n");
    return 0;
  }
  cloud.normals.resize(3, 0);  // clear input normals
  cloud.gridDownsample(0.005f);

  cilantro::Timer timer;
  timer.start();
  cilantro::KDTree3f<> tree(cloud.points);
  cilantro::NormalEstimation<float, 3, cilantro::MinimumCovarianceDeterminant<float, 3>> ne(tree);
  ne.setViewPoint(cilantro::Vector3f(0.f, 0.f, 0.f));
  ne.covarianceMethod().setChiSquareThreshold(6.25).setNumberOfTrials(2).setNumberOfRefinements(1).setSeed(7);
  cloud.normals = ne.getNormalsKNN(12);
  const size_t before = cloud.size();
  cloud.removeInvalidNormals();
  timer.stop();

  std::printf("Estimation time: %.3f ms\n", timer.getElapsedTime());
  std::printf("%zu points, %zu invalid normals, %zu kept\n", before, before - cloud.size(), cloud.size());
  return 0;
}
