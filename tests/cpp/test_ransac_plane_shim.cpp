// The plane-RANSAC shim (include/cilantro/model_estimation/ransac_hyperplane_estimator.hpp) and the PointCloud3f
// index-subset constructor and remove() (b200_shims.hpp). tests/test_ransac_plane_shims.py builds and runs it.
//
//   test_ransac_plane_shim <points.bin> <seed>
// points.bin: packed float32 xyz. Prints one line per result ("key values..."); floats as their bit patterns.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <cilantro/model_estimation/ransac_hyperplane_estimator.hpp>
#include <cilantro/utilities/point_cloud.hpp>

static void print_plane(const char* key, const cilantro::Hyperplane3f& h) {
  std::printf("%s", key);
  for (float c : h.coeffs()) {
    uint32_t u;
    std::memcpy(&u, &c, 4);
    std::printf(" %u", u);
  }
  std::printf("\n");
}

template <class V>
static void print_list(const char* key, const V& v) {
  std::printf("%s %zu", key, v.size());
  for (auto x : v) std::printf(" %llu", (unsigned long long)x);
  std::printf("\n");
}

static void print_points(const char* key, const cilantro::VectorSet3f& p) {
  std::printf("%s %zu", key, p.cols());
  for (size_t i = 0; i < 3 * p.cols(); i++) std::printf(" %g", p.data()[i]);
  std::printf("\n");
}

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  std::vector<float> xyz;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 3;
  float b[3];
  while (std::fread(b, sizeof(float), 3, f) == 3) xyz.insert(xyz.end(), b, b + 3);
  std::fclose(f);
  const uint32_t seed = (uint32_t)std::atoi(argv[2]);
  cilantro::PointCloud3f cloud;
  cloud.points.resize(3, xyz.size() / 3);
  std::memcpy(cloud.points.data(), xyz.data(), xyz.size() * sizeof(float));

  // the reference example's recipe (examples/ransac_plane_estimator.cpp)
  cilantro::PlaneRANSACEstimator3f<> pe(cloud.points);
  pe.setMaxInlierResidual(0.01f)
      .setTargetInlierCount((size_t)(0.15 * cloud.size()))
      .setMaxNumberOfIterations(250)
      .setReEstimationStep(false)
      .setRandomSeed(seed);
  const cilantro::Hyperplane3f plane = pe.estimate().getModel();
  std::printf("iterations %zu\ninliers %zu\n", pe.getNumberOfPerformedIterations(), pe.getNumberOfInliers());
  print_plane("plane", plane);
  print_list("inlier_list", pe.getModelInliers());
  const std::vector<float> r = pe.computeResiduals(plane);
  size_t k = 0;
  for (size_t i = 0; i < r.size(); i++) k += r[i] <= 0.01f ? 1 : 0;
  std::printf("recount %zu\n", k);
  print_plane("model_all", pe.estimateModel());
  print_plane("model_subset", pe.estimateModel(std::vector<size_t>{0, 5, 9, 13, 21, 40}));

  // index subsets and remove() on a small cloud with normals
  cilantro::PointCloud3f small;
  small.points.resize(3, 8);
  small.normals.resize(3, 8);
  for (size_t i = 0; i < 8; i++) {
    small.points.setCol(i, cilantro::Vector3f((float)i, 0.f, 0.f));
    small.normals.setCol(i, cilantro::Vector3f(0.f, (float)i, 0.f));
  }
  const std::vector<int> idx = {5, 1, 5, 3};
  print_points("subset", cilantro::PointCloud3f(small, idx).points);
  print_points("subset_normals", cilantro::PointCloud3f(small, idx).normals);
  print_points("negate", cilantro::PointCloud3f(small, idx, true).points);
  cilantro::PointCloud3f rem = small;
  rem.remove(std::vector<int>{1, 6, 1, 3});
  print_points("remove", rem.points);
  print_points("remove_normals", rem.normals);
  cilantro::PointCloud3f cut(cloud, pe.getModelInliers(), true);
  std::printf("cut %zu\n", cut.size());
  std::printf("all plane-RANSAC shim checks ran\n");
  return 0;
}
