// Example: the flow of cilantro's examples/rigid_icp.cpp and examples/normal_estimation.cpp — load, voxel-grid
// downsample, estimate normals, register with the combined-metric ICP, save — written against the cilantro names and
// running on an H100 through libcilantro_b200.so (no Eigen, no visualisation).
//
//   make -C examples && ./examples/register_clouds dst.ply src.ply [bin_size] [max_correspondence_distance]
//
// Without arguments a synthetic surface is generated, perturbed by a known pose and registered back.
#include <cilantro/registration/icp_common_instances.hpp>
#include <cilantro/utilities/point_cloud.hpp>
#include <cilantro/utilities/timer.hpp>

#include <cstdio>
#include <cstdlib>
#include <random>

static cilantro::PointCloud3f synthetic_surface(size_t n, unsigned seed) {
  std::mt19937 rng(seed);
  std::uniform_real_distribution<float> U(-1.f, 1.f);
  cilantro::PointCloud3f pc;
  pc.points.resize(3, n);
  for (size_t i = 0; i < n; i++) {
    const float u = U(rng), v = U(rng);
    pc.points.setCol(i, {u, v, 0.25f * std::sin(2.5f * u) * std::cos(2.f * v)});
  }
  return pc;
}

int main(int argc, char** argv) {
  cilantro::PointCloud3f dst, src;
  cilantro::RigidTransform3f pose;  // identity unless synthetic
  if (argc >= 3) {
    dst = cilantro::PointCloud3f(argv[1]);
    src = cilantro::PointCloud3f(argv[2]);
  } else {
    dst = synthetic_surface(400000, 1);
    src = dst;
    const float a = 0.04f;  // small rotation about z plus a shift
    pose.linear(0, 0) = std::cos(a); pose.linear(0, 1) = -std::sin(a);
    pose.linear(1, 0) = std::sin(a); pose.linear(1, 1) = std::cos(a);
    pose.translation(0) = 0.02f; pose.translation(1) = -0.01f; pose.translation(2) = 0.015f;
    src.transform(pose);
  }
  if (dst.isEmpty() || src.isEmpty()) {
    std::printf("empty input cloud\n");
    return 1;
  }
  const float bin = argc >= 4 ? (float)std::atof(argv[3]) : 0.01f;
  const float max_dist = argc >= 5 ? (float)std::atof(argv[4]) : 0.1f;

  cilantro::Timer timer;
  timer.start();
  dst.gridDownsample(bin);
  src.gridDownsample(bin);
  dst.estimateNormalsKNN(10);  // view point = origin, like PointCloud::estimateNormalsKNN
  timer.stop();
  std::printf("downsample + normals: %zu / %zu points, %.2f ms\n", dst.size(), src.size(), timer.getElapsedTime());

  timer.start();
  cilantro::SimpleCombinedMetricRigidICP3f icp(dst.points, dst.normals, src.points);
  icp.setMaxNumberOfOptimizationStepIterations(1).setPointToPointMetricWeight(0.1f).setPointToPlaneMetricWeight(1.0f);
  icp.correspondenceSearchEngine().setMaxDistance(max_dist * max_dist);
  icp.setConvergenceTolerance(1e-5f).setMaxNumberOfIterations(50);
  const cilantro::RigidTransform3f T = icp.estimate().getTransform();
  timer.stop();
  std::printf("ICP: %zu iterations, converged %d, %.2f ms\n", icp.getNumberOfPerformedIterations(), (int)icp.hasConverged(),
              timer.getElapsedTime());
  for (int r = 0; r < 3; r++)
    std::printf("  [% .6f % .6f % .6f | % .6f]\n", T.linear(r, 0), T.linear(r, 1), T.linear(r, 2), T.translation(r));
  if (argc < 3) {
    const cilantro::RigidTransform3f back = T * pose;  // should be the identity
    float err = 0.f;
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) err += (back.linear(r, c) - (r == c)) * (back.linear(r, c) - (r == c));
      err += back.translation(r) * back.translation(r);
    }
    std::printf("|T * pose - I|_F = %.2e\n", std::sqrt(err));
    if (!(std::sqrt(err) < 1e-2f)) return 2;
  }
  src.transform(T);
  src.toPLYFile("registered.ply");
  std::printf("wrote registered.ply\n");
  return 0;
}
