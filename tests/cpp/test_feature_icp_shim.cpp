// C++ surface of the feature-space ICP (tests/test_feature_icp_shims.py): the reference example's engine-templated call
// sequence over the drop-in headers. Input: a raw float32 file holding dst, dst normals, dst colours, src, src normals,
// src colours (n x 3 each); argv: path n_dst n_src. Prints one line per run: name, the 12 transform words as uint32,
// iterations, correspondences.
#include <cilantro/correspondence_search/common_transformable_feature_adaptors.hpp>
#include <cilantro/correspondence_search/correspondence_search_kd_tree.hpp>
#include <cilantro/registration/icp_common_instances.hpp>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

static void print(const char* name, const cilantro::RigidTransform3f& T, size_t iters, size_t corr) {
  std::printf("%s", name);
  for (int i = 0; i < 12; i++) {
    uint32_t b;
    std::memcpy(&b, T.data() + i, 4);
    std::printf(" %u", b);
  }
  std::printf(" %zu %zu\n", iters, corr);
}

template <class ICP>
static void setup(ICP& icp) {
  icp.setMaxNumberOfOptimizationStepIterations(1).setPointToPointMetricWeight(0.1f).setPointToPlaneMetricWeight(1.0f);
  icp.correspondenceSearchEngine().setMaxDistance(0.05f);
  icp.setConvergenceTolerance(0.f).setMaxNumberOfIterations(10);
}

int main(int argc, char** argv) {
  if (argc < 4) return 1;
  const size_t nd = std::strtoul(argv[2], nullptr, 10), ns = std::strtoul(argv[3], nullptr, 10);
  std::vector<float> buf(3 * (3 * nd + 3 * ns));
  FILE* f = std::fopen(argv[1], "rb");
  if (!f || std::fread(buf.data(), sizeof(float), buf.size(), f) != buf.size()) return 1;
  std::fclose(f);
  const float* p = buf.data();
  cilantro::ConstVectorSetMatrixMap3f dp(p, nd), dn(p + 3 * nd, nd), dc(p + 6 * nd, nd);
  p += 9 * nd;
  cilantro::ConstVectorSetMatrixMap3f sp(p, ns), sn(p + 3 * ns, ns), sc(p + 6 * ns, ns);
  cilantro::DistanceEvaluator<float> dist_eval;
  cilantro::UnityWeightEvaluator<float> w;

  {  // the reference example's recipe
    cilantro::PointNormalColorFeaturesAdaptor3f dst_feat(dp, dn, dc, 0.5, 5.0);
    cilantro::PointNormalColorFeaturesAdaptor3f src_feat(sp, sn, sc, 0.5, 5.0);
    cilantro::CorrespondenceSearchKDTree<decltype(dst_feat)> engine(dst_feat, src_feat, dist_eval);
    cilantro::CombinedMetricRigidTransformICP3f<decltype(engine)> icp(dp, dn, sp, engine, w, w);
    setup(icp);
    icp.estimate();
    print("feat", icp.getTransform(), icp.getNumberOfPerformedIterations(), icp.getCorrespondences().size());
    if (engine.getCorrespondences().size() != icp.getCorrespondences().size()) return 3;
  }
  {  // PointFeaturesAdaptor3f engine and the Simple... class
    cilantro::PointFeaturesAdaptor3f dst_feat(dp), src_feat(sp);
    cilantro::CorrespondenceSearchKDTree<decltype(dst_feat)> engine(dst_feat, src_feat, dist_eval);
    cilantro::CombinedMetricRigidTransformICP3f<decltype(engine)> icp(dp, dn, sp, engine, w, w);
    setup(icp);
    icp.estimate();
    print("point", icp.getTransform(), icp.getNumberOfPerformedIterations(), icp.getCorrespondences().size());
    cilantro::SimpleCombinedMetricRigidICP3f simple(dp, dn, sp);
    setup(simple);
    simple.estimate();
    print("simple", simple.getTransform(), simple.getNumberOfPerformedIterations(), simple.getCorrespondences().size());
  }
  {  // point-to-point over colour features: from (points, colours, weight) and from the pre-assembled 6 x N matrix
    cilantro::PointColorFeaturesAdaptor3f dst_feat(dp, dc, 5.0), src_feat(sp, sc, 5.0);
    std::vector<float> dm(6 * nd), sm(6 * ns);
    for (size_t i = 0; i < nd; i++)
      for (int k = 0; k < 3; k++) dm[6 * i + k] = dp.data()[3 * i + k], dm[6 * i + 3 + k] = 5.0f * dc.data()[3 * i + k];
    for (size_t i = 0; i < ns; i++)
      for (int k = 0; k < 3; k++) sm[6 * i + k] = sp.data()[3 * i + k], sm[6 * i + 3 + k] = 5.0f * sc.data()[3 * i + k];
    cilantro::PointColorFeaturesAdaptor3f dst_pre(dm), src_pre(sm);
    for (int pre = 0; pre < 2; pre++) {
      auto& a = pre ? dst_pre : dst_feat;
      auto& b = pre ? src_pre : src_feat;
      cilantro::CorrespondenceSearchKDTree<cilantro::PointColorFeaturesAdaptor3f> engine(a, b, dist_eval);
      cilantro::PointToPointMetricRigidTransformICP3f<decltype(engine)> icp(dp, sp, engine);
      icp.correspondenceSearchEngine().setMaxDistance(0.05f).setSearchDirection(cilantro::CorrespondenceSearchDirection::BOTH);
      icp.setConvergenceTolerance(0.f).setMaxNumberOfIterations(6);
      icp.estimate();
      print(pre ? "color_pre" : "color", icp.getTransform(), icp.getNumberOfPerformedIterations(),
            icp.getCorrespondences().size());
    }
  }
  return 0;
}
