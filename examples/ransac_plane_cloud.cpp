// Plane RANSAC through the shims: PLY (or a synthetic room corner) -> gridDownsample -> PlaneRANSACEstimator3f with the
// recipe of the reference's examples/ransac_plane_estimator.cpp -> cut the plane out of the cloud.
//   make -C examples ransac_plane_cloud && ./examples/ransac_plane_cloud [cloud.ply]
#include <cmath>
#include <cstdio>
#include <random>

#include <cilantro/model_estimation/ransac_hyperplane_estimator.hpp>
#include <cilantro/utilities/point_cloud.hpp>

int main(int argc, char** argv) {
  cilantro::PointCloud3f cloud;
  if (argc > 1) {
    cloud = cilantro::PointCloud3f(argv[1]);
  } else {  // a floor (z = 0, 60 %) and clutter above it (40 %)
    std::mt19937 rng(1);
    std::uniform_real_distribution<float> u(0.f, 4.f);
    std::normal_distribution<float> noise(0.f, 0.002f);
    const size_t n = 200000;
    cloud.points.resize(3, n);
    for (size_t i = 0; i < n; i++)
      cloud.points.setCol(i, i % 5 < 3 ? cilantro::Vector3f(u(rng), u(rng), noise(rng))
                                       : cilantro::Vector3f(u(rng), u(rng), 0.2f + 0.5f * u(rng)));
  }
  if (cloud.isEmpty()) {
    std::printf("Input cloud is empty!\n");
    return 0;
  }
  cloud.gridDownsample(0.01f);

  cilantro::PlaneRANSACEstimator3f<> pe(cloud.points);
  pe.setMaxInlierResidual(0.01f)
      .setTargetInlierCount((size_t)(0.15 * cloud.size()))
      .setMaxNumberOfIterations(250)
      .setReEstimationStep(true);
  const cilantro::Hyperplane3f plane = pe.estimate().getModel();
  const auto& inliers = pe.getModelInliers();
  std::printf("RANSAC iterations: %zu, inlier count: %zu\n", pe.getNumberOfPerformedIterations(), pe.getNumberOfInliers());
  std::printf("plane: %.5f %.5f %.5f %.5f\n", plane.normal()[0], plane.normal()[1], plane.normal()[2], plane.offset());

  const cilantro::PointCloud3f rest(cloud, inliers, true);  // everything but the plane
  std::printf("%zu points -> %zu on the plane, %zu left\n", cloud.size(), inliers.size(), rest.size());
  return 0;
}
