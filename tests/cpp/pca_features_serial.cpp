// Serial C++ restatement of the PCA projection and reconstruction folds (DESIGN §4.18), for pinning the numpy
// restatement tests/pca_features_ref.py on the CPU. Compiled with -ffp-contract=off: every fp32 operation rounds once.
//
//   pca_features_serial in.bin out.bin
//   in:  int64 n, D, k; float32 rows [n x D]; float32 mean [D]; float32 evecs [D x D] (row-major, columns = basis);
//        float32 q [n x k]
//   out: float32 projection [n x k]; float32 reconstruction of q [n x D]
#include <cstdint>
#include <cstdio>
#include <vector>

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  int64_t hdr[3];
  if (std::fread(hdr, sizeof(int64_t), 3, f) != 3) return 2;
  const int64_t n = hdr[0], D = hdr[1], k = hdr[2];
  std::vector<float> rows(n * D), mean(D), E(D * D), q(n * k);
  if (std::fread(rows.data(), sizeof(float), rows.size(), f) != rows.size()) return 2;
  if (std::fread(mean.data(), sizeof(float), mean.size(), f) != mean.size()) return 2;
  if (std::fread(E.data(), sizeof(float), E.size(), f) != E.size()) return 2;
  if (std::fread(q.data(), sizeof(float), q.size(), f) != q.size()) return 2;
  std::fclose(f);

  std::vector<float> proj(n * k), rec(n * D);
  for (int64_t i = 0; i < n; i++) {
    // project(points, k), principal_component_analysis.hpp:46-50
    for (int64_t j = 0; j < k; j++) {
      float acc = 0.f;
      for (int64_t d = 0; d < D; d++) {
        const float c = rows[i * D + d] - mean[d];
        acc = acc + E[d * D + j] * c;
      }
      proj[i * k + j] = acc;
    }
    // reconstruct(points), :59-62
    for (int64_t r = 0; r < D; r++) {
      float acc = 0.f;
      for (int64_t j = 0; j < k; j++) acc = acc + E[r * D + j] * q[i * k + j];
      rec[i * D + r] = acc + mean[r];
    }
  }
  FILE* o = std::fopen(argv[2], "wb");
  if (!o) return 2;
  std::fwrite(proj.data(), sizeof(float), proj.size(), o);
  std::fwrite(rec.data(), sizeof(float), rec.size(), o);
  std::fclose(o);
  return 0;
}
