// Serial C++ restatement of k-means over D-dimensional rows (DESIGN §4.17), for pinning the numpy restatement
// tests/kmeans_features_ref.py on the CPU. Compiled with -ffp-contract=off: every fp32 operation rounds once.
//
//   kmeans_features_serial in.bin out.bin
//   in:  int64 n, D, k, max_iter; float32 tol; float32 rows [n x D]; float32 centroids [k x D]
//   out: int64 iterations; float32 centroids [k x D]; int64 labels [n]; int64 labels of the first assignment [n]
//
// The loop is the reference's brute-force branch (clustering/kmeans.hpp:67-194) with the per-cluster sums and counts
// in double over the rows whose components are all finite, the fp32 division sum * (1 / count), and the empty-cluster
// repair from the largest cluster's farthest finite member (ties to the lowest index).
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <limits>
#include <vector>

static float fold_d2(const float* c, const float* p, int64_t D) {
  float acc = 0.f;
  for (int64_t j = D - 1; j >= 0; j--) {
    const float d = c[j] - p[j];
    acc = d * d + acc;
  }
  return acc;
}

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  int64_t hdr[4];
  float tol;
  if (std::fread(hdr, sizeof(int64_t), 4, f) != 4 || std::fread(&tol, sizeof(float), 1, f) != 1) return 2;
  const int64_t n = hdr[0], D = hdr[1], k = hdr[2], max_iter = hdr[3];
  std::vector<float> pts(n * D), cent(k * D);
  if (std::fread(pts.data(), sizeof(float), pts.size(), f) != pts.size()) return 2;
  if (std::fread(cent.data(), sizeof(float), cent.size(), f) != cent.size()) return 2;
  std::fclose(f);

  std::vector<char> finite(n, 1);
  for (int64_t i = 0; i < n; i++)
    for (int64_t j = 0; j < D; j++)
      if (!std::isfinite(pts[i * D + j])) finite[i] = 0;

  std::vector<int64_t> labels(n, 0), first;
  std::vector<float> old;
  const float tol_sq = tol * tol;
  int64_t it = 0;
  while (it < max_iter) {
    bool changed = false;
    for (int64_t i = 0; i < n; i++) {  // :100-119
      float best = std::numeric_limits<float>::infinity();
      int64_t bi = 0;
      for (int64_t j = 0; j < k; j++) {
        const float d = fold_d2(&cent[j * D], &pts[i * D], D);
        if (d < best) {
          best = d;
          bi = j;
        }
      }
      if (labels[i] != bi) changed = true;
      labels[i] = bi;
    }
    if (first.empty()) first = labels;
    if (!changed && it > 0) break;  // :122
    old = cent;
    std::vector<double> s(k * D, 0.0), cnt(k, 0.0);
    for (int64_t i = 0; i < n; i++) {
      if (!finite[i]) continue;
      for (int64_t j = 0; j < D; j++) s[labels[i] * D + j] += (double)pts[i * D + j];
      cnt[labels[i]] += 1.0;
    }
    std::vector<float> oc(D);
    for (int64_t i = 0; i < k; i++) {  // :134-176
      if (cnt[i] != 0.0) continue;
      int64_t max_ind = 0;
      for (int64_t j = 1; j < k; j++)
        if (cnt[j] > cnt[max_ind]) max_ind = j;
      const float inv = 1.0f / (float)cnt[max_ind];
      for (int64_t r = 0; r < D; r++) oc[r] = (float)s[max_ind * D + r] * inv;
      int64_t far = -1;
      float far_d = -1.f;
      for (int64_t m = 0; m < n; m++) {
        if (labels[m] != max_ind || !finite[m]) continue;
        const float d = fold_d2(oc.data(), &pts[m * D], D);
        if (d > far_d) {
          far_d = d;
          far = m;
        }
      }
      if (far < 0) continue;
      labels[far] = i;
      for (int64_t r = 0; r < D; r++) s[max_ind * D + r] -= (double)pts[far * D + r];
      cnt[max_ind] -= 1.0;
      cnt[i] += 1.0;
    }
    for (int64_t j = 0; j < k; j++) {  // :179-181
      const float inv = 1.0f / (float)cnt[j];
      for (int64_t r = 0; r < D; r++) cent[j * D + r] = (float)s[j * D + r] * inv;
    }
    it++;
    if (tol > 0.f) {  // :186-188
      float mx = 0.f;
      for (int64_t j = 0; j < k; j++) {
        const float v = fold_d2(&cent[j * D], &old[j * D], D);
        if (mx < v) mx = v;
      }
      if (mx < tol_sq) break;
    }
  }
  if (first.empty()) first.assign(n, 0);

  FILE* o = std::fopen(argv[2], "wb");
  if (!o) return 2;
  std::fwrite(&it, sizeof(int64_t), 1, o);
  std::fwrite(cent.data(), sizeof(float), cent.size(), o);
  std::fwrite(labels.data(), sizeof(int64_t), labels.size(), o);
  std::fwrite(first.data(), sizeof(int64_t), first.size(), o);
  std::fclose(o);
  return 0;
}
