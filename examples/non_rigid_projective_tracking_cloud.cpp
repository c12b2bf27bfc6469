// Non-rigid tracking of a deforming surface seen by a depth camera, on the device: a sheet 1 m in front of the camera
// is bent a little more in every frame and rendered into a 640 x 480 depth image with pointsToDepthImage; each frame is
// converted back to points with organised normals and tracked against the first frame's cloud with
// SimpleCombinedMetricSparseRigidWarpFieldProjectiveICP3f: control nodes from a 2.5 cm grid downsampling of the frame,
// 4-NN control lists, 8-NN node neighbourhoods and the sparse recipe of the reference's examples/non_rigid_icp.cpp,
// correspondences by projection into the first frame's image. Prints the mean point-to-plane residual of every frame
// before and after.
//   make -C examples non_rigid_projective_tracking_cloud && ./examples/non_rigid_projective_tracking_cloud
#include <cilantro/core/grid_downsampler.hpp>
#include <cilantro/core/image_point_cloud_conversions.hpp>
#include <cilantro/core/kd_tree.hpp>
#include <cilantro/registration/icp_common_instances.hpp>
#include <cilantro/utilities/point_cloud.hpp>

#include <cmath>
#include <cstdio>
#include <vector>

// frame k: a 0.8 x 0.6 m sheet with a fixed relief and a bend that grows with k, n x n samples (far more than pixels)
static cilantro::VectorSet3f sheet(int k, size_t n = 900) {
  cilantro::VectorSet3f p(3, n * n);
  for (size_t r = 0; r < n; r++)
    for (size_t c = 0; c < n; c++) {
      const float x = -0.4f + 0.8f * c / (n - 1), y = -0.3f + 0.6f * r / (n - 1);
      const float z = 1.f + 0.02f * std::sin(6.f * x) * std::cos(5.f * y) + 0.004f * k * (x / 0.4f) * (x / 0.4f) -
                      0.002f * k * (y / 0.3f);
      p.setCol(r * n + c, {x, y, z});
    }
  return p;
}

static float mean(const std::vector<float>& v) {
  double s = 0;
  for (float x : v) s += x;
  return v.empty() ? 0.f : (float)(s / v.size());
}

int main() {
  const size_t w = 640, h = 480;
  const cilantro::b200::Intrinsics3f K(525.f, 525.f, 319.5f, 239.5f);
  const cilantro::DepthValueConverter<float, float> conv(1.f);
  std::vector<float> depth(w * h);

  cilantro::pointsToDepthImage(sheet(0), K, conv, depth.data(), w, h);
  const cilantro::PointCloud3f model(depth.data(), conv, w, h, K, false, true);
  std::printf("model: %zu points with image normals\n", model.size());
  if (model.isEmpty()) return 1;

  const float control_res = 0.025f;
  float worst = 0.f;
  for (int k = 1; k <= 4; k++) {
    cilantro::pointsToDepthImage(sheet(k), K, conv, depth.data(), w, h);
    const cilantro::PointCloud3f frame(depth.data(), conv, w, h, K, false, true);
    cilantro::VectorSet<float, 3> control_points =
        cilantro::PointsGridDownsampler3f(frame.points, control_res).getDownsampledPoints();
    cilantro::KDTree<float, 3> control_tree(control_points);
    cilantro::NeighborhoodSet<float> src_to_control_nn =
        control_tree.search(frame.points, cilantro::KNNNeighborhoodSpecification<>(4));
    cilantro::NeighborhoodSet<float> regularization_nn =
        control_tree.search(control_points, cilantro::KNNNeighborhoodSpecification<>(8));

    cilantro::SimpleCombinedMetricSparseRigidWarpFieldProjectiveICP3f icp(
        model.points, model.normals, frame.points, src_to_control_nn, control_points.cols(), regularization_nn);
    icp.correspondenceSearchEngine().setProjectionIntrinsicMatrix(K).setProjectionImageWidth(w)
        .setProjectionImageHeight(h).setMaxDistance(0.02f * 0.02f);
    icp.controlWeightEvaluator().setSigma(0.5f * control_res);
    icp.regularizationWeightEvaluator().setSigma(3.0f * control_res);
    icp.setMaxNumberOfIterations(15).setConvergenceTolerance(2.5e-3f);
    icp.setMaxNumberOfGaussNewtonIterations(1).setGaussNewtonConvergenceTolerance(5e-4f);
    icp.setMaxNumberOfConjugateGradientIterations(500).setConjugateGradientConvergenceTolerance(1e-5f);
    icp.setPointToPointMetricWeight(0.0f).setPointToPlaneMetricWeight(1.0f).setStiffnessRegularizationWeight(200.0f);
    icp.setHuberLossBoundary(1e-2f);
    const float r0 = mean(icp.getResiduals());
    icp.estimate();
    const float r1 = mean(icp.getResiduals());
    worst = std::fmax(worst, r1 / r0);
    std::printf("frame %d: %zu points, %zu nodes, %zu iterations, %zu correspondences, mean residual %.3e -> %.3e\n", k,
                frame.size(), (size_t)control_points.cols(), icp.getNumberOfPerformedIterations(),
                icp.getCorrespondences().size(), r0, r1);
  }
  std::printf("worst residual ratio: %.3f\n", worst);
  return worst < 0.5f ? 0 : 2;
}
