// The projective ICP drop-ins (correspondence_search/correspondence_search_projective.hpp) run the fusion example's
// localisation call sequence; tests/test_projective_icp_shims.py compares each transform with the C ABI's bit for bit.
//
//   test_projective_icp_shim scene.bin
//
// scene.bin: u64 n_dst, n_src, w, h; f32 K[9] (row-major), E[12], T0[12] ([R | t] row-major); f32 dst[3 n_dst],
// dst_normals[3 n_dst], src[3 n_src], src_normals[3 n_src].
// Output, one line per run: name, the 12 transform entries as uint32 bit patterns, iterations, correspondences.
#include <cilantro/registration/icp_common_instances.hpp>

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

namespace {

template <class T>
T get(FILE* f) {
  T v;
  if (std::fread(&v, sizeof(T), 1, f) != 1) throw 1;
  return v;
}

cilantro::VectorSet3f cloud(FILE* f, size_t n) {
  cilantro::VectorSet3f s(3, n);
  if (n && std::fread(s.data(), sizeof(float), 3 * n, f) != 3 * n) throw 1;
  return s;
}

void print(const char* name, const cilantro::RigidTransform3f& T, size_t iters, size_t corr) {
  std::printf("%s", name);
  for (int i = 0; i < 12; i++) {
    uint32_t b;
    std::memcpy(&b, T.data() + i, 4);
    std::printf(" %u", b);
  }
  std::printf(" %zu %zu\n", iters, corr);
}

template <class Engine>
void configure(Engine& e, const cilantro::RigidTransform3f& E, const cilantro::b200::Intrinsics3f& K, size_t w, size_t h) {
  // the fusion example's setter chain
  e.setProjectionExtrinsicMatrix(E).setMaxDistance(0.1f * 0.1f).setProjectionImageWidth(w).setProjectionImageHeight(h)
      .setProjectionIntrinsicMatrix(K);
}

}  // namespace

int main(int argc, char** argv) {
  if (argc != 2) return 2;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  const size_t nd = get<uint64_t>(f), ns = get<uint64_t>(f), w = get<uint64_t>(f), h = get<uint64_t>(f);
  float k9[9], e12[12], t12[12];
  if (std::fread(k9, 4, 9, f) != 9 || std::fread(e12, 4, 12, f) != 12 || std::fread(t12, 4, 12, f) != 12) return 2;
  const cilantro::VectorSet3f dst = cloud(f, nd), dst_n = cloud(f, nd), src = cloud(f, ns), src_n = cloud(f, ns);
  std::fclose(f);
  const cilantro::b200::Intrinsics3f K(k9);
  const cilantro::RigidTransform3f E(e12), T0(t12);

  cilantro::SimpleCombinedMetricRigidProjectiveICP3f icp(dst, dst_n, src);
  configure(icp.correspondenceSearchEngine(), E, K, w, h);
  icp.setInitialTransform(T0).setConvergenceTolerance(5e-4f);
  icp.setMaxNumberOfIterations(6).setMaxNumberOfOptimizationStepIterations(1);
  icp.estimate();
  print("simple", icp.getTransform(), icp.getNumberOfPerformedIterations(), icp.getCorrespondences().size());
  // the same object again: the projection is already attached and must give the same result
  icp.estimate();
  print("again", icp.getTransform(), icp.getNumberOfPerformedIterations(), icp.getCorrespondences().size());
  // a setter re-attaches at the next estimate(): an image of width 0 has no correspondences
  icp.correspondenceSearchEngine().setProjectionImageWidth(0);
  icp.estimate();
  print("empty", icp.getTransform(), icp.getNumberOfPerformedIterations(), icp.getCorrespondences().size());

  cilantro::SimpleCombinedMetricRigidProjectiveICP3f sym(dst, dst_n, src, src_n);
  configure(sym.correspondenceSearchEngine(), E, K, w, h);
  sym.setInitialTransform(T0).setConvergenceTolerance(5e-4f);
  sym.setMaxNumberOfIterations(6).setMaxNumberOfOptimizationStepIterations(1);
  sym.estimate();
  print("symmetric", sym.getTransform(), sym.getNumberOfPerformedIterations(), sym.getCorrespondences().size());

  // PointToPointMetricRigidTransformICP3f over a caller-owned engine
  cilantro::PointFeaturesAdaptor3f dst_feat(dst), src_feat(src);
  cilantro::DistanceEvaluator<float, float> dist;
  cilantro::CorrespondenceSearchProjective<float> engine(dst_feat, src_feat, dist);
  configure(engine, E, K, w, h);
  cilantro::PointToPointMetricRigidTransformICP3f<cilantro::CorrespondenceSearchProjective<float>> p2p(dst, src, engine);
  p2p.setInitialTransform(T0).setConvergenceTolerance(5e-4f);
  p2p.setMaxNumberOfIterations(6);
  p2p.estimate();
  const size_t p2p_corr = p2p.getCorrespondences().size();
  if (engine.getCorrespondences().size() != p2p_corr) return 3;  // the engine holds the list, as the reference's does
  print("p2p", p2p.getTransform(), p2p.getNumberOfPerformedIterations(), p2p_corr);
  // the reference's defaults
  cilantro::CorrespondenceSearchProjective<float> fresh(dst_feat, src_feat, dist);
  const cilantro::b200::Intrinsics3f& Kd = fresh.getProjectionIntrinsicMatrix();
  const bool defaults = Kd(0, 0) == 528.f && Kd(1, 1) == 528.f && Kd(0, 2) == 320.f && Kd(1, 2) == 240.f && Kd(2, 2) == 1.f &&
                    Kd(0, 1) == 0.f && Kd(2, 0) == 0.f && fresh.getProjectionImageHeight() == 480 &&
                    fresh.getMaxDistance() == (float)(0.01 * 0.01) && fresh.getInlierFraction() == 1.0;
  std::printf("defaults %d\n", (int)(defaults && fresh.getProjectionImageWidth() == 640));
  return 0;
}
