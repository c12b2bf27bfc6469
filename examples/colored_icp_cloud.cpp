// Example: the coloured ICP recipe of cilantro's examples/rigid_icp.cpp (its commented "custom" block) — point + normal +
// colour feature adaptors as the correspondence search space of the combined-metric ICP — written against the cilantro
// names and running on an H100 through libcilantro_b200.so.
//
//   make -C examples colored_icp_cloud && ./examples/colored_icp_cloud [dst.ply src.ply] [bin_size]
//
// The PLYs need colours (normals are estimated when missing). Without arguments a low-relief sheet with a colour texture
// is generated and its second sample shifted in-plane: the geometry barely constrains that shift, the colours do.
#include <cilantro/correspondence_search/common_transformable_feature_adaptors.hpp>
#include <cilantro/correspondence_search/correspondence_search_kd_tree.hpp>
#include <cilantro/registration/icp_common_instances.hpp>
#include <cilantro/utilities/point_cloud.hpp>
#include <cilantro/utilities/timer.hpp>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>

static cilantro::PointCloud3f textured_sheet(size_t n, unsigned seed, float dx, float dy) {
  std::mt19937 rng(seed);
  std::uniform_real_distribution<float> U(0.f, 1.f);
  const float tau = 6.2831853f;
  cilantro::PointCloud3f pc;
  pc.points.resize(3, n);
  pc.colors.resize(3, n);
  for (size_t i = 0; i < n; i++) {
    const float x = U(rng), y = U(rng);
    pc.points.setCol(i, {x - dx, y - dy, 0.002f * std::sin(7 * x) * std::cos(6 * y)});
    pc.colors.setCol(i, {0.5f + 0.5f * std::sin(tau * 4 * x) * std::cos(tau * 3 * y),
                         0.5f + 0.5f * std::cos(tau * 5 * x + 1.f) * std::sin(tau * 3 * y + 0.5f),
                         0.5f + 0.5f * std::sin(tau * 3 * (x + y))});
  }
  return pc;
}

int main(int argc, char** argv) {
  const bool synthetic = argc < 3;
  const float dx = 0.03f, dy = -0.02f;
  cilantro::PointCloud3f dst, src;
  if (!synthetic) {
    dst = cilantro::PointCloud3f(argv[1]);
    src = cilantro::PointCloud3f(argv[2]);
  } else {
    dst = textured_sheet(200000, 1, 0.f, 0.f);
    src = textured_sheet(200000, 2, dx, dy);
  }
  if (dst.isEmpty() || src.isEmpty() || !dst.hasColors() || !src.hasColors()) {
    std::printf("input clouds must be non-empty and have colours\n");
    return 1;
  }
  const float bin = argc >= 4 ? (float)std::atof(argv[3]) : 0.005f;

  cilantro::Timer timer;
  timer.start();
  dst.gridDownsample(bin);
  src.gridDownsample(bin);
  if (!dst.hasNormals()) dst.estimateNormalsKNN(10);
  if (!src.hasNormals()) src.estimateNormalsKNN(10);
  timer.stop();
  std::printf("downsample + normals: %zu / %zu points, %.2f ms\n", dst.size(), src.size(), timer.getElapsedTime());

  timer.start();
  cilantro::PointNormalColorFeaturesAdaptor3f dst_feat(dst.points, dst.normals, dst.colors, 0.5, 5.0);
  cilantro::PointNormalColorFeaturesAdaptor3f src_feat(src.points, src.normals, src.colors, 0.5, 5.0);
  cilantro::DistanceEvaluator<float> dist_eval;
  cilantro::CorrespondenceSearchKDTree<decltype(dst_feat)> corr_engine(dst_feat, src_feat, dist_eval);
  cilantro::UnityWeightEvaluator<float> corr_weight_eval;
  cilantro::CombinedMetricRigidTransformICP3f<decltype(corr_engine)> icp(dst.points, dst.normals, src.points, corr_engine,
                                                                         corr_weight_eval, corr_weight_eval);
  icp.setMaxNumberOfOptimizationStepIterations(1).setPointToPointMetricWeight(0.1f).setPointToPlaneMetricWeight(1.0f);
  icp.correspondenceSearchEngine().setMaxDistance(0.1f * 0.1f);
  icp.setConvergenceTolerance(1e-5f).setMaxNumberOfIterations(30);
  const cilantro::RigidTransform3f T = icp.estimate().getTransform();
  timer.stop();
  std::printf("coloured ICP: %zu iterations, %zu correspondences, %.2f ms\n", icp.getNumberOfPerformedIterations(),
              icp.getCorrespondences().size(), timer.getElapsedTime());
  for (int r = 0; r < 3; r++)
    std::printf("  [% .6f % .6f % .6f | % .6f]\n", T.linear(r, 0), T.linear(r, 1), T.linear(r, 2), T.translation(r));
  if (synthetic) {
    const float ex = T.translation(0) - dx, ey = T.translation(1) - dy;
    const float err = std::sqrt(ex * ex + ey * ey);
    std::printf("in-plane offset error = %.2e\n", err);
    if (!(err < 5e-3f)) return 2;
  }
  src.transform(T);
  src.toPLYFile("colored_registered.ply");
  return 0;
}
