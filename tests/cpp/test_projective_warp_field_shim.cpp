// The projective warp-field drop-ins through the call sequence of examples/non_rigid_projective_tracking_cloud.cpp
// (tests/test_projective_warp_field_shims.py compares the output with the C ABI bit for bit). Input: the binary scene
// written by the test (sizes, K, dst, dst normals, src, the control lists and node neighbourhoods as CSRs). Output: a
// binary record per run (iterations, transforms, dense field, getCorrespondences()): the sparse class, the sparse class
// again after a width setter (re-attach), and the dense class with empty regularisation neighbourhoods.
#include <cilantro/registration/icp_common_instances.hpp>

#include <cstdint>
#include <cstdio>
#include <vector>

template <class T>
static std::vector<T> take(FILE* f, size_t n) {
  std::vector<T> v(n);
  if (n && std::fread(v.data(), sizeof(T), n, f) != n) throw std::runtime_error("short scene file");
  return v;
}

static std::vector<cilantro::NeighborSet<float, size_t>> lists(const std::vector<uint64_t>& off,
                                                              const std::vector<int64_t>& idx,
                                                              const std::vector<float>& val) {
  std::vector<cilantro::NeighborSet<float, size_t>> out(off.size() - 1);
  for (size_t j = 0; j + 1 < off.size(); j++)
    for (uint64_t k = off[j]; k < off[j + 1]; k++) out[j].push_back({(size_t)idx[k], val[k]});
  return out;
}

template <class Icp>
static void put(FILE* f, Icp& icp, const cilantro::TransformSet<cilantro::RigidTransform3f>& T,
                const cilantro::TransformSet<cilantro::RigidTransform3f>& Td) {
  const uint64_t it = icp.getNumberOfPerformedIterations();
  const auto& corr = icp.getCorrespondences();
  const uint64_t m = T.size(), n = Td.size(), c = corr.size();
  std::fwrite(&it, 8, 1, f);
  std::fwrite(&m, 8, 1, f);
  std::fwrite(&n, 8, 1, f);
  std::fwrite(&c, 8, 1, f);
  for (const auto& t : T) std::fwrite(t.data(), 4, 12, f);
  for (const auto& t : Td) std::fwrite(t.data(), 4, 12, f);
  for (const auto& p : corr) {
    const uint64_t a = p.indexInFirst, b = p.indexInSecond;
    std::fwrite(&a, 8, 1, f);
    std::fwrite(&b, 8, 1, f);
    std::fwrite(&p.value, 4, 1, f);
  }
}

int main(int argc, char** argv) {
  if (argc < 3) return 1;
  FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 1;
  const auto hdr = take<uint64_t>(in, 8);  // n_dst, n_src, m, ctrl entries, reg lists, reg entries, w, h
  const auto K9 = take<float>(in, 9);
  const auto dst = take<float>(in, 3 * hdr[0]), dst_n = take<float>(in, 3 * hdr[0]), src = take<float>(in, 3 * hdr[1]);
  const auto coff = take<uint64_t>(in, hdr[1] + 1);
  const auto cidx = take<int64_t>(in, hdr[3]);
  const auto cval = take<float>(in, hdr[3]);
  const auto roff = take<uint64_t>(in, hdr[4] + 1);
  const auto ridx = take<int64_t>(in, hdr[5]);
  const auto rval = take<float>(in, hdr[5]);
  std::fclose(in);
  const size_t w = hdr[6], h = hdr[7], m = hdr[2];
  const cilantro::b200::Intrinsics3f K(K9.data());
  const cilantro::ConstVectorSetMatrixMap3f D(dst), DN(dst_n), S(src);
  FILE* out = std::fopen(argv[2], "wb");
  if (!out) return 1;

  cilantro::SimpleCombinedMetricSparseRigidWarpFieldProjectiveICP3f icp(D, DN, S, lists(coff, cidx, cval), m,
                                                                        lists(roff, ridx, rval));
  icp.correspondenceSearchEngine().setProjectionIntrinsicMatrix(K).setProjectionImageWidth(w)
      .setProjectionImageHeight(h).setMaxDistance(0.02f * 0.02f);
  icp.controlWeightEvaluator().setSigma(0.5f * 0.025f);
  icp.regularizationWeightEvaluator().setSigma(3.0f * 0.025f);
  icp.setMaxNumberOfIterations(15).setConvergenceTolerance(2.5e-3f);
  icp.setMaxNumberOfGaussNewtonIterations(1).setGaussNewtonConvergenceTolerance(5e-4f);
  icp.setMaxNumberOfConjugateGradientIterations(500).setConjugateGradientConvergenceTolerance(1e-5f);
  icp.setPointToPointMetricWeight(0.0f).setPointToPlaneMetricWeight(1.0f).setStiffnessRegularizationWeight(200.0f);
  icp.setHuberLossBoundary(1e-2f);
  icp.estimate();
  put(out, icp, icp.getTransform(), icp.getDenseWarpField());
  // the engine's own getter holds the list the ICP's getter read
  if (icp.correspondenceSearchEngine().getCorrespondences().size() != icp.getCorrespondences().size()) return 3;
  icp.correspondenceSearchEngine().setProjectionImageWidth(w - 8);
  icp.estimate();
  put(out, icp, icp.getTransform(), icp.getDenseWarpField());

  std::vector<cilantro::NeighborSet<float, size_t>> none;
  cilantro::SimpleCombinedMetricDenseRigidWarpFieldProjectiveICP3f dense(D, DN, S, none);
  dense.correspondenceSearchEngine().setProjectionIntrinsicMatrix(K).setProjectionImageWidth(w)
      .setProjectionImageHeight(h).setMaxDistance(0.04f * 0.04f);
  dense.setMaxNumberOfIterations(3).setMaxNumberOfGaussNewtonIterations(1).setPointToPointMetricWeight(0.1f);
  dense.setStiffnessRegularizationWeight(200.0f).setMaxNumberOfConjugateGradientIterations(500);
  dense.estimate();
  put(out, dense, dense.getTransform(), dense.getTransform());
  std::fclose(out);
  std::printf("projective warp-field shim runs written\n");
  return 0;
}
