// The reference's examples/mean_shift.cpp recipe on the device: a synthetic cloud of three Gaussian blobs, every point
// a seed, kernel radius 2 sigma, cluster tolerance 0.2 sigma, through the MeanShift3f shim (cb_cloud_mean_shift).
// Build: make -C examples mean_shift_cloud (after python -m cilantro_b200.build). Prints the modes.
#include <cilantro/clustering/mean_shift.hpp>

#include <chrono>
#include <cstdio>
#include <random>

int main() {
  const float sigma = 0.1f;
  const float centres[3][3] = {{0.f, 0.f, 0.f}, {1.f, 0.f, 0.f}, {0.f, 1.f, 1.f}};
  const size_t per_blob = 2000;
  cilantro::VectorSet3f pts(3, 3 * per_blob);
  std::mt19937 rng(7);
  std::normal_distribution<float> g(0.f, sigma);
  for (size_t b = 0; b < 3; b++)
    for (size_t j = 0; j < per_blob; j++)
      pts.setCol(b * per_blob + j, {centres[b][0] + g(rng), centres[b][1] + g(rng), centres[b][2] + g(rng)});

  cilantro::MeanShift3f<> ms(pts);
  const auto t0 = std::chrono::steady_clock::now();
  ms.cluster(2.f * sigma, 5000, 0.2f * sigma);
  const double ms_taken = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  std::printf("%zu seeds, %zu iterations, %.1f ms\n", pts.cols(), ms.getNumberOfPerformedIterations(), ms_taken);
  for (size_t c = 0; c < ms.getNumberOfClusters(); c++) {
    const auto m = ms.getClusterModes().col(c);
    std::printf("cluster %zu: %zu seeds, mode (%.4f, %.4f, %.4f)\n", c, ms.getClusterToPointIndicesMap()[c].size(), m[0],
                m[1], m[2]);
  }
  std::printf("%zu clusters found\n", ms.getNumberOfClusters());
  return 0;
}
