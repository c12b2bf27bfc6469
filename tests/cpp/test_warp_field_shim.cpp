// C++ drop-in test of SimpleCombinedMetricDenseRigidWarpFieldICP3f (registration/icp_common_instances.hpp): the
// reference example's dense recipe through the class's setters, the inherited ICP surface, TransformSet /
// transformPoints / PointCloud3f::transformed and the rejected inputs, running on the GPU through libcilantro_b200.so.
// Exit code 0 = all checks passed. Built and run by tests/test_gpu_warp_field.py.
#include <cilantro/core/kd_tree.hpp>
#include <cilantro/registration/icp_common_instances.hpp>
#include <cilantro/utilities/point_cloud.hpp>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>

#define CHECK(cond)                                                          \
  do {                                                                       \
    if (!(cond)) {                                                           \
      std::printf("CHECK failed at %s:%d: %s\n", __FILE__, __LINE__, #cond); \
      return 1;                                                              \
    }                                                                        \
  } while (0)

static double mean(const std::vector<float>& v) {
  double s = 0;
  for (float x : v) s += x;
  return v.empty() ? 0.0 : s / v.size();
}

int main() {
  // a 60 x 60 grid at 5 mm on a smooth height field; the source is the same grid bent by up to 6 mm
  const int side = 60;
  const float h = 0.005f, k = 2.f * 3.14159265f / (side * h);
  cilantro::PointCloud3f dst, src;
  dst.points.resize(3, side * side);
  src.points.resize(3, side * side);
  for (int i = 0; i < side; i++)
    for (int j = 0; j < side; j++) {
      const float x = i * h, y = j * h, z = 0.02f * std::sin(0.5f * k * x) * std::cos(0.5f * k * y);
      dst.points.setCol(i * side + j, {x, y, z});
      src.points.setCol(i * side + j, {x + 0.004f * std::sin(k * y), y + 0.002f, z + 0.004f * std::cos(k * x)});
    }
  dst.estimateNormalsKNN(12);
  CHECK(dst.hasNormals());
  const auto nbhd = cilantro::KDTree3f<>(src.points).search(src.points, cilantro::KNNNeighborhoodSpecification<>(12));

  cilantro::SimpleCombinedMetricDenseRigidWarpFieldICP3f icp(dst.points, dst.normals, src.points, nbhd);
  // defaults of CombinedMetricDenseWarpFieldICP and IterativeClosestPointBase
  CHECK(icp.getPointToPointMetricWeight() == 0.f && icp.getPointToPlaneMetricWeight() == 1.f);
  CHECK(icp.getStiffnessRegularizationWeight() == 1.f && icp.getHuberLossBoundary() == 1e-4f);
  CHECK(icp.getMaxNumberOfGaussNewtonIterations() == 10 && icp.getMaxNumberOfConjugateGradientIterations() == 1000);
  CHECK(icp.getGaussNewtonConvergenceTolerance() == 1e-5f && icp.getConjugateGradientConvergenceTolerance() == 1e-5f);
  CHECK(icp.getMaxNumberOfIterations() == 15 && icp.getConvergenceTolerance() == 1e-5f);
  CHECK(icp.getInitialTransform().size() == src.size() && !icp.hasConverged());

  icp.correspondenceSearchEngine().setMaxDistance(0.02f * 0.02f);
  icp.regularizationWeightEvaluator().setSigma(3.f * h);
  icp.setMaxNumberOfIterations(15).setConvergenceTolerance(2.5e-3f);
  icp.setMaxNumberOfGaussNewtonIterations(1).setGaussNewtonConvergenceTolerance(5e-4f);
  icp.setMaxNumberOfConjugateGradientIterations(500).setConjugateGradientConvergenceTolerance(1e-5f);
  icp.setPointToPointMetricWeight(0.1f).setPointToPlaneMetricWeight(1.0f).setStiffnessRegularizationWeight(200.0f);
  icp.setHuberLossBoundary(1e-2f);
  CHECK(icp.getMaxNumberOfGaussNewtonIterations() == 1 && icp.getHuberLossBoundary() == 1e-2f);

  const double r0 = mean(icp.getResiduals());
  const cilantro::TransformSet<cilantro::RigidTransform3f> tf = icp.estimate().getTransform();
  const double r1 = mean(icp.getResiduals());
  std::printf("iterations %zu, converged %d, last update %.3e, residual %.3e -> %.3e\n",
              icp.getNumberOfPerformedIterations(), (int)icp.hasConverged(), icp.getLastUpdateNorm(), r0, r1);
  CHECK(tf.size() == src.size());
  CHECK(icp.getNumberOfPerformedIterations() >= 1 && icp.getNumberOfPerformedIterations() <= 15);
  CHECK(icp.hasConverged() == (icp.getLastUpdateNorm() < icp.getConvergenceTolerance()));
  CHECK(r1 < r0);
  // the shim forwards every setting: the same call through the C ABI gives the same transforms, bit for bit
  {
    cb_context* ctx = cilantro::b200::Context::get();  // the shims' context (one per process and device)
    cb_cloud *cd = nullptr, *cs = nullptr;
    CHECK(cb_cloud_create(ctx, dst.points.data(), dst.normals.data(), dst.size(), 0, &cd) == CB_OK);
    CHECK(cb_cloud_create(ctx, src.points.data(), nullptr, src.size(), 0, &cs) == CB_OK);
    std::vector<uint64_t> off(1, 0);
    std::vector<int64_t> idx;
    std::vector<float> val;
    for (const auto& list : nbhd) {
      for (const auto& nb : list) {
        idx.push_back((int64_t)nb.index);
        val.push_back(nb.value);
      }
      off.push_back(idx.size());
    }
    cb_warp_icp* w = nullptr;
    CHECK(cb_warp_icp_create(ctx, cd, cs, off.data(), idx.data(), val.data(), nbhd.size(), &w) == CB_OK);
    cb_warp_params prm;
    cb_warp_default_params(&prm);
    prm.max_d2 = 0.02f * 0.02f;
    prm.reg_coeff = -0.5f / ((3.f * h) * (3.f * h));
    prm.max_iter = 15;
    prm.tol = 2.5e-3f;
    prm.max_gn_iter = 1;
    prm.gn_tol = 5e-4f;
    prm.max_cg_iter = 500;
    prm.cg_tol = 1e-5f;
    prm.w_pt = 0.1f;
    prm.w_pl = 1.0f;
    prm.stiffness = 200.0f;
    prm.huber = 1e-2f;
    std::vector<float> T(12 * src.size());
    cb_warp_result res;
    CHECK(cb_warp_icp_estimate(w, &prm, nullptr, T.data(), &res) == CB_OK);
    CHECK((size_t)res.iterations == icp.getNumberOfPerformedIterations());
    for (size_t i = 0; i < src.size(); i++) CHECK(std::memcmp(&T[12 * i], tf[i].data(), 12 * sizeof(float)) == 0);
    cb_warp_icp_destroy(w);
    cb_cloud_destroy(cd);
    cb_cloud_destroy(cs);
  }
  const auto& corr = icp.getCorrespondences();
  CHECK(!corr.empty() && corr.size() <= src.size());
  for (size_t c = 1; c < corr.size(); c++) CHECK(corr[c].indexInSecond > corr[c - 1].indexInSecond);

  // every per-point transform is a rotation
  for (const auto& T : tf) {
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) {
        float d = 0.f;
        for (int r = 0; r < 3; r++) d += T.linear(r, a) * T.linear(r, b);
        CHECK(std::fabs(d - (a == b ? 1.f : 0.f)) < 1e-5f);
      }
  }
  // transformPoints over the set, and PointCloud3f::transformed
  cilantro::VectorSet3f warped;
  cilantro::transformPoints(tf, src.points, warped);
  const cilantro::PointCloud3f src_t = src.transformed(tf);
  CHECK(warped.cols() == src.size() && src_t.size() == src.size());
  for (size_t i = 0; i < src.size(); i += 97) {
    const cilantro::Vector3f q = tf[i] * src.points.col(i);
    for (int r = 0; r < 3; r++) CHECK(warped(r, i) == q[r] && src_t.points(r, i) == q[r]);
  }

  // starting from the estimate, one more iteration moves little
  icp.setInitialTransform(tf);
  icp.estimate(1, 0.f);
  CHECK(icp.getNumberOfPerformedIterations() == 1 && icp.getLastUpdateNorm() < 0.05f);

  // rejected inputs: a wrong-sized initial transform set, point-to-plane without destination normals
  bool threw = false;
  icp.setInitialTransform(cilantro::TransformSet<cilantro::RigidTransform3f>(3));
  try {
    icp.estimate();
  } catch (const std::runtime_error&) {
    threw = true;
  }
  CHECK(threw);
  cilantro::SimpleCombinedMetricDenseRigidWarpFieldICP3f no_normals(dst.points, cilantro::VectorSet3f(), src.points, nbhd);
  threw = false;
  try {
    no_normals.estimate();
  } catch (const std::runtime_error&) {
    threw = true;
  }
  CHECK(threw);
  no_normals.setPointToPlaneMetricWeight(0.f).setPointToPointMetricWeight(1.f).setMaxNumberOfIterations(2);
  no_normals.correspondenceSearchEngine().setMaxDistance(0.02f * 0.02f);
  CHECK(no_normals.estimate().getTransform().size() == src.size());
  std::printf("all warp-field shim checks passed\n");
  return 0;
}
