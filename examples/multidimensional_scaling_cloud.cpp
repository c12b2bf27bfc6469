// Example: classical multidimensional scaling of the wavy ring (cos t, sin t, 0.1 sin 10 t), 1000 points, into the plane
// with MultidimensionalScaling<float, 2>, written against the cilantro names and running on an H100 through
// libcilantro_b200.so: the eigenvalues, the embedding dimension and the stress of the embedding.
//
//   make -C examples multidimensional_scaling_cloud && ./examples/multidimensional_scaling_cloud
#include <cilantro/utilities/multidimensional_scaling.hpp>
#include <cilantro/utilities/timer.hpp>

#include <cmath>
#include <cstdio>
#include <vector>

struct SquareMatrix {  // n x n column-major floats: data(), rows(), cols(), as an Eigen::MatrixXf
  size_t n = 0;
  std::vector<float> d;
  float& operator()(size_t i, size_t j) { return d[j * n + i]; }
  float operator()(size_t i, size_t j) const { return d[j * n + i]; }
  const float* data() const { return d.data(); }
  size_t rows() const { return n; }
  size_t cols() const { return n; }
};

int main() {
  const size_t n = 1000;
  const float pi = 3.14159265358979323846f;
  std::vector<float> p(3 * n);
  for (size_t i = 0; i < n; i++) {
    const float t = (2.0f * pi * i) / n;
    p[3 * i] = std::cos(t);
    p[3 * i + 1] = std::sin(t);
    p[3 * i + 2] = 0.1f * std::sin(10.0f * t);
  }
  SquareMatrix dist_sq{n, std::vector<float>(n * n)};
  for (size_t i = 0; i < n; i++)
    for (size_t j = 0; j < n; j++) {
      float s = 0.f;
      for (int k = 0; k < 3; k++) s += (p[3 * i + k] - p[3 * j + k]) * (p[3 * i + k] - p[3 * j + k]);
      dist_sq(i, j) = s;
    }
  std::printf("Number of points: %zu\n", n);

  cilantro::Timer timer;
  timer.start();
  const cilantro::MultidimensionalScaling<float, 2> mds(dist_sq);
  timer.stop();
  std::printf("Elapsed time: %.3f ms\n", timer.getElapsedTime());

  const auto& ev = mds.getComputedEigenValues();
  std::printf("Eigenvalues:");
  for (size_t i = 0; i < ev.rows(); i++) std::printf(" %.6g", ev[i]);
  std::printf("\nEmbedding dimension: %zu\n", mds.getEmbeddingDimension());

  // Kruskal's stress-1 of the embedded distances against the input distances
  const auto& e = mds.getEmbeddedPoints();
  const size_t dim = e.rows();
  double num = 0.0, den = 0.0;
  for (size_t i = 0; i < n; i++)
    for (size_t j = i + 1; j < n; j++) {
      double s = 0.0;
      for (size_t k = 0; k < dim; k++) s += ((double)e(k, i) - e(k, j)) * ((double)e(k, i) - e(k, j));
      const double d_in = std::sqrt((double)dist_sq(i, j)), d_out = std::sqrt(s);
      num += (d_in - d_out) * (d_in - d_out);
      den += d_in * d_in;
    }
  std::printf("Stress: %.6g\n", std::sqrt(num / den));
  return 0;
}
