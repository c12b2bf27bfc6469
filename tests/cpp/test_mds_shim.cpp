// The C++ drop-in of multidimensional scaling (MultidimensionalScaling<float, D>, computeDistancePreservingSpectralEmbedding,
// estimateEmbeddingDimensionEigengap), run on the device; tests/test_mds_shims.py compares the output with the C ABI
// through capi bit for bit.
//
//   test_mds_shim in.bin out.bin
//   in:  int64 n, max_dim, estimate_dim, squared; float32 distances [n x n] column-major
//   out: int64 nev, dim, eigengap dim; float32 eigenvalues [nev], embedding [dim x n] column-major, all of
//        MultidimensionalScalingXf; then the same two arrays of computeDistancePreservingSpectralEmbedding (none when it
//        throws std::invalid_argument) and, when
//        max_dim is 2 or 3 without estimation, of MultidimensionalScaling2f / 3f
#include <cilantro/utilities/multidimensional_scaling.hpp>

#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <vector>

struct ColMajor {  // a column-major float matrix of the kind the drop-in takes
  size_t n;
  std::vector<float> d;
  const float* data() const { return d.data(); }
  size_t rows() const { return n; }
  size_t cols() const { return n; }
};

template <class E, class V>
static void put(FILE* o, const E& ev, const V& emb) {
  std::fwrite(ev.data(), sizeof(float), ev.rows(), o);
  std::fwrite(emb.data(), sizeof(float), emb.rows() * emb.cols(), o);
}

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  int64_t hdr[4];
  if (std::fread(hdr, sizeof(int64_t), 4, f) != 4) return 2;
  const size_t n = (size_t)hdr[0], max_dim = (size_t)hdr[1];
  const bool est = hdr[2] != 0, sq = hdr[3] != 0;
  ColMajor m{n, std::vector<float>(n * n)};
  if (std::fread(m.d.data(), sizeof(float), n * n, f) != n * n) return 2;
  std::fclose(f);
  FILE* o = std::fopen(argv[2], "wb");
  if (!o) return 2;
  const cilantro::MultidimensionalScalingXf x(m, max_dim, est, sq);
  const int64_t sizes[3] = {(int64_t)x.getComputedEigenValues().rows(), (int64_t)x.getEmbeddingDimension(),
                            (int64_t)cilantro::estimateEmbeddingDimensionEigengap(x.getComputedEigenValues(), max_dim)};
  std::fwrite(sizes, sizeof(int64_t), 3, o);
  put(o, x.getComputedEigenValues(), x.getEmbeddedPoints());
  cilantro::VectorSet<float, cilantro::b200::kDynamic> emb;
  cilantro::b200::DenseMatrixF<cilantro::b200::kDynamic, 1> ev;
  try {  // max_dim = 0 without estimation is the eigen-solver's argument error
    cilantro::computeDistancePreservingSpectralEmbedding<float>(m, max_dim, est, sq, emb, ev);
    put(o, ev, emb);
  } catch (const std::invalid_argument&) {
  }
  if (!est && max_dim == 2) {
    const cilantro::MultidimensionalScaling2f y(m, sq);
    put(o, y.getComputedEigenValues(), y.getEmbeddedPoints());
  } else if (!est && max_dim == 3) {
    const cilantro::MultidimensionalScaling3f y(m, sq);
    put(o, y.getComputedEigenValues(), y.getEmbeddedPoints());
  }
  std::fclose(o);
  return 0;
}
