// Example: PCA of per-point features [p, w_n n, w_c c] (9-D) with PrincipalComponentAnalysis<float, 9>, written against
// the cilantro names and running on an H100 through libcilantro_b200.so: the explained-variance ratios, then the
// features projected to 3-D on the device.
//
//   make -C examples pca_features_cloud && ./examples/pca_features_cloud [cloud.ply] [w_n] [w_c]
//
// The PLY needs colours. Without arguments a flat sheet with a colour texture is generated and its normals estimated.
#include <cilantro/core/principal_component_analysis.hpp>
#include <cilantro/utilities/point_cloud.hpp>
#include <cilantro/utilities/timer.hpp>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>

static cilantro::PointCloud3f textured_sheet(size_t n, unsigned seed) {
  std::mt19937 rng(seed);
  std::uniform_real_distribution<float> U(0.f, 1.f);
  const float tau = 6.2831853f;
  cilantro::PointCloud3f pc;
  pc.points.resize(3, n);
  pc.colors.resize(3, n);
  for (size_t i = 0; i < n; i++) {
    const float x = U(rng), y = U(rng);
    pc.points.setCol(i, {x, y, 0.02f * std::sin(7 * x) * std::cos(6 * y)});
    const float stripe = std::sin(tau * 4 * x) * std::cos(tau * 3 * y) > 0.f ? 1.f : 0.f;
    pc.colors.setCol(i, {stripe, 0.5f + 0.5f * std::sin(tau * 3 * (x + y)), 1.f - stripe});
  }
  return pc;
}

int main(int argc, char** argv) {
  cilantro::PointCloud3f cloud = argc >= 2 ? cilantro::PointCloud3f(argv[1]) : textured_sheet(200000, 1);
  if (cloud.isEmpty() || !cloud.hasColors()) {
    std::printf("input cloud must be non-empty and have colours\n");
    return 1;
  }
  const float w_n = argc >= 3 ? (float)std::atof(argv[2]) : 0.1f;
  const float w_c = argc >= 4 ? (float)std::atof(argv[3]) : 0.15f;
  if (!cloud.hasNormals()) cloud.estimateNormalsKNN(10);

  const size_t n = cloud.points.cols();
  cilantro::VectorSet<float, 9> features(9, n);
  for (size_t i = 0; i < n; i++)
    for (size_t r = 0; r < 3; r++) {
      features(r, i) = cloud.points(r, i);
      features(3 + r, i) = w_n * cloud.normals(r, i);
      features(6 + r, i) = w_c * cloud.colors(r, i);
    }

  cilantro::Timer timer;
  timer.start();
  cilantro::PrincipalComponentAnalysis<float, 9> pca(features);
  const cilantro::VectorSet<float, 3> low = pca.project<3>(features);
  timer.stop();

  const auto& ev = pca.getEigenValues();
  double total = 0;
  for (int j = 0; j < 9; j++) total += ev.data()[j];
  std::printf("PCA<float, 9>: %zu points, %.1f ms (PCA + projection to 3-D), explained variance", n,
              timer.getElapsedTime());
  for (int j = 0; j < 9; j++) std::printf(" %.3f", total > 0 ? ev.data()[j] / total : 0.0);
  std::printf("\nfirst projected point: (%.4f, %.4f, %.4f)\n", low(0, 0), low(1, 0), low(2, 0));
  return 0;
}
