// Example: colour-aware k-means, the 6-D recipe cilantro's examples/kmeans.cpp keeps in a comment — each point's
// [p; 0.15 c] clustered with KMeans<float, 6, KDTreeDistanceAdaptors::L2> — written against the cilantro names and
// running on an H100 through libcilantro_b200.so.
//
//   make -C examples colored_kmeans_cloud && ./examples/colored_kmeans_cloud [cloud.ply] [k] [bin_size]
//
// The PLY needs colours. Without arguments a flat sheet with a colour texture is generated: the xyz alone would cut it
// into similar patches, the colour term pulls the cluster borders towards the texture's edges.
#include <cilantro/clustering/kmeans.hpp>
#include <cilantro/utilities/point_cloud.hpp>
#include <cilantro/utilities/timer.hpp>

#include <algorithm>
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
    pc.points.setCol(i, {x, y, 0.002f * std::sin(7 * x) * std::cos(6 * y)});
    const float stripe = std::sin(tau * 4 * x) * std::cos(tau * 3 * y) > 0.f ? 1.f : 0.f;
    pc.colors.setCol(i, {stripe, 0.5f + 0.5f * std::sin(tau * 3 * (x + y)), 1.f - stripe});
  }
  return pc;
}

int main(int argc, char** argv) {
  cilantro::PointCloud3f cloud = argc >= 2 ? cilantro::PointCloud3f(argv[1]) : textured_sheet(400000, 1);
  if (cloud.isEmpty() || !cloud.hasColors()) {
    std::printf("input cloud must be non-empty and have colours\n");
    return 1;
  }
  const size_t k = argc >= 3 ? (size_t)std::atol(argv[2]) : 250;
  const float bin = argc >= 4 ? (float)std::atof(argv[3]) : 0.005f;
  cloud.gridDownsample(bin);

  // data_points.topRows(3) = points; data_points.bottomRows(3) = 0.15 * colors
  const size_t n = cloud.points.cols();
  cilantro::VectorSet<float, 6> data_points(6, n);
  for (size_t i = 0; i < n; i++)
    for (size_t r = 0; r < 3; r++) {
      data_points(r, i) = cloud.points(r, i);
      data_points(3 + r, i) = 0.15f * cloud.colors(r, i);
    }

  cilantro::KMeans<float, 6, cilantro::KDTreeDistanceAdaptors::L2> kmc(data_points);
  cilantro::Timer timer;
  timer.start();
  kmc.cluster(k, 100, std::numeric_limits<float>::epsilon(), true, 1u);
  timer.stop();

  const auto& lists = kmc.getClusterToPointIndicesMap();
  size_t mins = n, maxs = 0;
  for (const auto& l : lists) {
    mins = std::min(mins, l.size());
    maxs = std::max(maxs, l.size());
  }
  std::printf("colored k-means: %zu points, k = %zu, %zu iterations in %.1f ms, cluster sizes %zu..%zu\n", n,
              kmc.getNumberOfClusters(), kmc.getNumberOfPerformedIterations(), timer.getElapsedTime(), mins, maxs);
  return 0;
}
