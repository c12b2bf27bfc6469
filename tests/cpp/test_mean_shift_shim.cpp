// C++ drop-in test of clustering/mean_shift.hpp: the reference's calls (both constructors, both cluster() overloads,
// both kernel evaluators, the getters and the ClusteringBase maps) on a known answer, running on the GPU through
// libcilantro_b200.so. Exit code 0 = all checks passed. Built and run by tests/test_gpu_mean_shift.py.
#include <cilantro/clustering/mean_shift.hpp>
#include <cilantro/core/kd_tree.hpp>

#include <cmath>
#include <cstdio>

#define CHECK(cond)                                                          \
  do {                                                                       \
    if (!(cond)) {                                                           \
      std::printf("CHECK failed at %s:%d: %s\n", __FILE__, __LINE__, #cond); \
      return 1;                                                              \
    }                                                                        \
  } while (0)

int main() {
  // two symmetric 7-point stars (centre + 6 axis neighbours at distance 0.1) around (0,0,0) and (5,0,0)
  cilantro::VectorSet3f pts(3, 14);
  const float d[7][3] = {{0, 0, 0}, {0.1f, 0, 0}, {-0.1f, 0, 0}, {0, 0.1f, 0}, {0, -0.1f, 0}, {0, 0, 0.1f}, {0, 0, -0.1f}};
  for (int b = 0; b < 2; b++)
    for (int j = 0; j < 7; j++) pts.setCol(7 * b + j, {5.f * b + d[j][0], d[j][1], d[j][2]});

  cilantro::MeanShift3f<> ms(pts);
  ms.cluster(0.5f, 100, 0.05f);  // all points as seeds, flat kernel
  CHECK(ms.getNumberOfClusters() == 2 && ms.getNumberOfPoints() == 14);
  CHECK(ms.getShiftedSeeds().cols() == 14 && ms.getClusterModes().cols() == 2);
  CHECK(std::fabs(ms.getClusterModes().col(1)[0] - 5.f) < 1e-5f && std::fabs(ms.getClusterModes().col(0)[0]) < 1e-5f);
  CHECK(ms.getClusterToPointIndicesMap()[0].size() == 7 && ms.getClusterToPointIndicesMap()[1][0] == 7);
  CHECK(ms.getPointToClusterIndexMap()[13] == 1 && ms.getNumberOfPerformedIterations() >= 1);

  cilantro::KDTree3f<> tree(pts);
  cilantro::MeanShift3f<> from_tree(tree);
  cilantro::VectorSet3f seeds(3, 3);
  seeds.setCol(0, {4.8f, 0.f, 0.f});
  seeds.setCol(1, {0.2f, 0.f, 0.f});
  seeds.setCol(2, {50.f, 0.f, 0.f});  // no neighbours: NaN, its own cluster
  from_tree.cluster(seeds, 0.5f, 20, 0.05f, 1e-6f, cilantro::RBFKernelWeightEvaluator<float, float, true>(0.3f));
  CHECK(from_tree.getNumberOfClusters() == 3 && from_tree.getNumberOfPerformedIterations() == 20);
  CHECK(std::fabs(from_tree.getShiftedSeeds().col(0)[0] - 5.f) < 1e-4f && std::isnan(from_tree.getShiftedSeeds().col(2)[0]));
  from_tree.cluster(seeds, 0.5f, 0, 1.f);  // max_iter 0: the seeds as given, clustered
  CHECK(from_tree.getNumberOfPerformedIterations() == 0 && from_tree.getShiftedSeeds().col(1)[0] == 0.2f);
  CHECK(from_tree.getNumberOfClusters() == 3);
  std::printf("all mean-shift shim checks passed\n");
  return 0;
}
