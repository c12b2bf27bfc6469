// Non-rigid registration through the shims, the sparse recipe of the reference's examples/non_rigid_icp.cpp: control
// nodes from a 2.5 cm grid downsampling of the full-resolution source, 4-NN control lists and 8-NN node
// neighbourhoods, then SimpleCombinedMetricSparseRigidWarpFieldICP3f (one rigid transform per control node, blended
// onto every source point).
//   make -C examples sparse_non_rigid_icp_cloud && ./examples/sparse_non_rigid_icp_cloud [dst.ply src.ply]
// Without arguments it registers a synthetic pair: a smooth height field and a copy of it bent by 1 cm.
#include <cmath>
#include <cstdio>
#include <random>

#include <cilantro/core/grid_downsampler.hpp>
#include <cilantro/core/kd_tree.hpp>
#include <cilantro/registration/icp_common_instances.hpp>
#include <cilantro/utilities/point_cloud.hpp>
#include <cilantro/utilities/timer.hpp>

static float mean(const std::vector<float>& v) {
  double s = 0;
  for (float x : v) s += x;
  return v.empty() ? 0.f : (float)(s / v.size());
}

int main(int argc, char** argv) {
  cilantro::PointCloud3f dst, src;
  if (argc > 2) {
    dst = cilantro::PointCloud3f(argv[1]);
    src = cilantro::PointCloud3f(argv[2]);
  } else {  // 1 m x 1 m height field; the source is the same surface bent by a smooth 1 cm field and shifted
    std::mt19937 rng(1);
    std::uniform_real_distribution<float> u(0.f, 1.f);
    const size_t n = 120000;
    const float k = 2.f * 3.14159265f;
    dst.points.resize(3, n);
    src.points.resize(3, n);
    for (size_t i = 0; i < n; i++) {
      const float x = u(rng), y = u(rng), z = 0.08f * std::sin(0.5f * k * x) * std::cos(0.5f * k * y);
      dst.points.setCol(i, {x, y, z});
      src.points.setCol(i, {x + 0.01f * std::sin(k * x) + 0.003f, y + 0.01f * std::cos(k * y) - 0.003f,
                            z + 0.01f * std::sin(k * (x + y)) + 0.0015f});
    }
  }
  if (dst.isEmpty() || src.isEmpty()) {
    std::printf("Input cloud is empty!\n");
    return 0;
  }
  if (!dst.hasNormals()) dst.estimateNormalsKNN(12);

  const float control_res = 0.025f;
  cilantro::VectorSet<float, 3> control_points =
      cilantro::PointsGridDownsampler3f(src.points, control_res).getDownsampledPoints();
  cilantro::KDTree<float, 3> control_tree(control_points);
  cilantro::NeighborhoodSet<float> src_to_control_nn =
      control_tree.search(src.points, cilantro::KNNNeighborhoodSpecification<>(4));
  cilantro::NeighborhoodSet<float> regularization_nn =
      control_tree.search(control_points, cilantro::KNNNeighborhoodSpecification<>(8));

  cilantro::Timer timer;
  timer.start();
  cilantro::SimpleCombinedMetricSparseRigidWarpFieldICP3f icp(dst.points, dst.normals, src.points, src_to_control_nn,
                                                               control_points.cols(), regularization_nn);
  icp.correspondenceSearchEngine().setMaxDistance(0.02f * 0.02f);
  icp.controlWeightEvaluator().setSigma(0.5f * control_res);
  icp.regularizationWeightEvaluator().setSigma(3.0f * control_res);
  icp.setMaxNumberOfIterations(15).setConvergenceTolerance(2.5e-3f);
  icp.setMaxNumberOfGaussNewtonIterations(1).setGaussNewtonConvergenceTolerance(5e-4f);
  icp.setMaxNumberOfConjugateGradientIterations(500).setConjugateGradientConvergenceTolerance(1e-5f);
  icp.setPointToPointMetricWeight(0.0f).setPointToPlaneMetricWeight(1.0f).setStiffnessRegularizationWeight(200.0f);
  icp.setHuberLossBoundary(1e-2f);
  const float r0 = mean(icp.getResiduals());
  const auto tf_est = icp.estimate().getDenseWarpField();
  timer.stop();
  const float r1 = mean(icp.getResiduals());

  const cilantro::PointCloud3f src_trans = src.transformed(tf_est);
  std::printf("%zu source points, %zu control nodes -> %zu destination points\n", src.size(),
              (size_t)control_points.cols(), dst.size());
  std::printf("Registration time: %.1f ms\n", timer.getElapsedTime());
  std::printf("Iterations performed: %zu\n", icp.getNumberOfPerformedIterations());
  std::printf("Has converged: %d\n", (int)icp.hasConverged());
  std::printf("mean residual %.3e -> %.3e\n", r0, r1);
  std::printf("warped %zu points\n", src_trans.size());
  return 0;
}
