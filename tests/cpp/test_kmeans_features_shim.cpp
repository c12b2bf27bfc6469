// KMeans<float, 6>, KMeans3f<>, KMeansXf<> and KMeans2f<> (include/cilantro/b200_shims.hpp) on rows read from a file,
// for comparison with the C ABI's results (tests/test_kmeans_features_shims.py), and on empty sets.
//
//   test_kmeans_features_shim in.bin out.bin
//   in:  int64 n, D, k, max_iter, seed; float32 tol; float32 rows [n x D]; float32 centroids [k x D]
//   out: for cluster(centroids, ...) then cluster(k, ..., seed): int64 iterations; float32 centroids [k x D];
//        int64 labels [n]
#include <cilantro/clustering/kmeans.hpp>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <type_traits>
#include <vector>

// the reference's alias (clustering/kmeans.hpp:205-207): the distance adaptor first, then the index types
static_assert(std::is_same<cilantro::KMeans3f<>, cilantro::KMeans<float, 3>>::value, "KMeans3f<> is KMeans<float, 3>");

template <class KM, class Map>
static void run(FILE* o, const Map& data, const Map& cent, size_t k, size_t max_iter, float tol, uint32_t seed) {
  KM km(data);
  for (int pass = 0; pass < 2; pass++) {
    if (pass == 0)
      km.cluster(cent, max_iter, tol);
    else
      km.cluster(k, max_iter, tol, false, seed);
    const int64_t it = (int64_t)km.getNumberOfPerformedIterations();
    std::fwrite(&it, sizeof(it), 1, o);
    const auto& c = km.getClusterCentroids();
    std::fwrite(c.data(), sizeof(float), c.rows() * c.cols(), o);
    for (auto l : km.getPointToClusterIndexMap()) {
      const int64_t v = (int64_t)l;
      std::fwrite(&v, sizeof(v), 1, o);
    }
    size_t total = 0;
    for (const auto& m : km.getClusterToPointIndicesMap()) total += m.size();
    if (total != km.getNumberOfPoints() || km.getNumberOfClusters() != k) std::fprintf(stderr, "inconsistent maps\n");
  }
}

// An empty set (its data() may be null) in every dimension: one iteration in which every cluster is empty, so every
// centroid is 0 * (1 / 0) = NaN, no labels and k empty member lists.
template <class KM, class Set>
static bool empty_set_clusters_to_nothing(const Set& cent) {
  const Set empty;
  KM km(empty);
  km.cluster(cent, 10, 0.f);
  const auto& c = km.getClusterCentroids();
  bool ok = km.getNumberOfPerformedIterations() == 1 && km.getNumberOfPoints() == 0 && km.getNumberOfClusters() == 3;
  for (size_t i = 0; i < c.rows() * c.cols(); i++) ok = ok && std::isnan(c.data()[i]);
  for (const auto& m : km.getClusterToPointIndicesMap()) ok = ok && m.empty();
  return ok;
}

static bool empty_sets_cluster_to_nothing() {
  cilantro::VectorSet<float, 2> c2(2, 3);
  cilantro::VectorSet3f c3(3, 3);
  const bool ok = empty_set_clusters_to_nothing<cilantro::KMeans2f<>>(c2) &&
                  empty_set_clusters_to_nothing<cilantro::KMeans3f<>>(c3);
  if (!ok) std::fprintf(stderr, "k-means on an empty set\n");
  return ok;
}

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  int64_t h[5];
  float tol;
  if (std::fread(h, sizeof(int64_t), 5, f) != 5 || std::fread(&tol, sizeof(float), 1, f) != 1) return 2;
  const size_t n = h[0], D = h[1], k = h[2], max_iter = h[3];
  const uint32_t seed = (uint32_t)h[4];
  std::vector<float> rows(n * D), cent(k * D);
  if (std::fread(rows.data(), sizeof(float), rows.size(), f) != rows.size()) return 2;
  if (std::fread(cent.data(), sizeof(float), cent.size(), f) != cent.size()) return 2;
  std::fclose(f);
  FILE* o = std::fopen(argv[2], "wb");
  if (!o) return 2;
  if (D == 6) {
    using Map = cilantro::ConstVectorSetMatrixMap<float, 6>;
    run<cilantro::KMeans<float, 6, cilantro::KDTreeDistanceAdaptors::L2>>(o, Map(rows.data(), n), Map(cent.data(), k),
                                                                           k, max_iter, tol, seed);
  } else if (D == 3) {
    using Map = cilantro::ConstVectorSetMatrixMap<float, 3>;
    run<cilantro::KMeans3f<cilantro::KDTreeDistanceAdaptors::L2>>(o, Map(rows.data(), n), Map(cent.data(), k), k,
                                                                   max_iter, tol, seed);
  } else if (D == 2) {
    using Map = cilantro::ConstVectorSetMatrixMap<float, 2>;
    run<cilantro::KMeans2f<cilantro::KDTreeDistanceAdaptors::L2Simple>>(o, Map(rows.data(), n), Map(cent.data(), k),
                                                                         k, max_iter, tol, seed);
  } else {
    using Map = cilantro::ConstVectorSetMatrixMap<float, -1>;
    run<cilantro::KMeansXf<>>(o, Map(rows.data(), D, n), Map(cent.data(), D, k), k, max_iter, tol, seed);
  }
  std::fclose(o);
  if (!empty_sets_cluster_to_nothing()) return 1;
  std::printf("k-means shim: D = %zu done\n", D);
  return 0;
}
