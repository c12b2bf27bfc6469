// Host check of cilantro_b200/csrc/mcd_rule.hpp (the pinned rule of the robust normal estimation), compiled with
// -ffp-contract=off:
//   * minstd_seed / minstd_next equal std::minstd_rand0, and uniform_below(n) equals
//     std::uniform_int_distribution<size_t>(0, n - 1) on it, for n = 1..256 over many seeds (the installed libstdc++);
//   * point_seed spreads neighbouring indices (no two equal seeds among the first 2^20 indices of one user seed);
//   * sort_key orders NaN and +inf last (ties by position), -inf first, negative keys below zero, -0 as +0, and
//     agrees with the float order everywhere else;
//   * subset_size follows llround, including negative and overflowing products;
//   * determinant and inverse agree with float64 on well-conditioned matrices: |det - det64| <= 8 eps |det|-scale,
//     |A inv(A) - I| <= 64 eps cond.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <limits>
#include <random>
#include <unordered_set>
#include <vector>

#include "mcd_rule.hpp"

using namespace cb::mcd;

static int failures = 0;
#define CHECK(cond, ...)            \
  do {                              \
    if (!(cond)) {                  \
      std::printf("FAIL: " __VA_ARGS__); \
      std::printf("\n");            \
      failures++;                   \
    }                               \
  } while (0)

int main() {
  // generator and draws
  std::mt19937 seeds(7);
  long draws = 0;
  const uint32_t edge_seeds[4] = {0u, 1u, 2147483647u, 4294967295u};
  for (int trial = 0; trial < 400; trial++) {
    const uint32_t s = trial < 4 ? edge_seeds[trial] : (uint32_t)seeds();
    std::minstd_rand0 ref(s);
    uint32_t x = minstd_seed(s);
    for (int i = 0; i < 50; i++) CHECK((uint32_t)ref() == minstd_next(x), "minstd seed %u step %d", s, i);
    for (uint32_t n = 1; n <= 256; n++) {
      std::minstd_rand0 g(s);
      std::uniform_int_distribution<size_t> dist(0, n - 1);
      uint32_t y = minstd_seed(s);
      for (int i = 0; i < 20; i++, draws++) {
        const size_t want = dist(g);
        const uint32_t got = uniform_below(y, n);
        if (want != got) {
          CHECK(false, "uniform n=%u seed %u draw %d: %zu vs %u", n, s, i, want, got);
          break;
        }
      }
    }
  }
  std::printf("generator: %ld draws equal to libstdc++\n", draws);
  {
    std::unordered_set<uint32_t> seen;
    for (uint32_t i = 0; i < (1u << 20); i++) seen.insert(point_seed(12345u, i));
    CHECK(seen.size() == (1u << 20), "point_seed collisions: %zu distinct", seen.size());
  }

  // key order
  const float inf = std::numeric_limits<float>::infinity(), nan = std::numeric_limits<float>::quiet_NaN();
  CHECK(sort_key(nan, 0) > sort_key(3e38f, 9) && sort_key(nan, 0) < sort_key(inf, 5), "NaN with +inf, after finite");
  CHECK(sort_key(nan, 3) > sort_key(nan, 2) && sort_key(inf, 2) < sort_key(nan, 3), "NaN ties by position");
  CHECK(key_bits(nan) == key_bits(inf), "NaN sorts as +inf");
  CHECK(sort_key(-inf, 9) < sort_key(-1e30f, 0), "-inf first");
  CHECK(sort_key(-1.f, 9) < sort_key(0.f, 0), "negative keys below zero");
  CHECK(key_bits(-0.f) == key_bits(0.f), "-0 as +0");
  CHECK(sort_key(2.f, 1) < sort_key(2.f, 2) && sort_key(2.f, 2) < sort_key(std::nextafter(2.f, 3.f), 0), "ties");
  {
    std::mt19937 r(3);
    std::uniform_real_distribution<float> u(-1.f, 1.f);
    for (int i = 0; i < 1000000; i++) {
      const float a = u(r) * std::ldexp(1.f, (int)(r() % 200) - 100), b = u(r) * std::ldexp(1.f, (int)(r() % 200) - 100);
      CHECK((a < b) == (key_bits(a) < key_bits(b)), "key order %g %g", a, b);
      if (failures > 20) break;
    }
  }

  // h
  CHECK(subset_size(0.75f, 12, 3) == 9, "h 0.75*12");
  CHECK(subset_size(0.5f, 5, 3) == 3, "h 2.5 rounds away from zero, then max(min)");  // llround(2.5) = 3
  CHECK(subset_size(0.5f, 7, 3) == 4, "h 3.5 -> 4");
  CHECK(subset_size(1.0f, 12, 3) == 12 && subset_size(2.0f, 12, 3) == 12, "h capped at size");
  CHECK(subset_size(0.0f, 12, 3) == 3 && subset_size(-0.01f, 12, 3) == 3, "h small ratio -> min");
  CHECK(subset_size(-1.0f, 12, 3) == 12, "h negative llround wraps to size");
  CHECK(subset_size(3e38f, 128, 3) == 128, "h overflowing product -> size");
  for (uint32_t size = 4; size <= 128; size++)
    for (float ratio : {0.1f, 0.3f, 0.5f, 0.6f, 0.75f, 0.9f, 0.99f}) {
      const long long r = std::llround(ratio * (float)size);
      const size_t want = std::min(std::max((size_t)3, (size_t)r), (size_t)size);
      CHECK(subset_size(ratio, size, 3) == want, "h ratio %g size %u", ratio, size);
    }

  // 3x3 algebra against float64
  {
    std::mt19937 r(11);
    std::normal_distribution<double> nd;
    double worst_det = 0, worst_inv = 0;
    for (int t = 0; t < 100000; t++) {
      // A = Q diag(l) Q^T, eigenvalues in [1, 10] times a scale: condition <= 10
      double l[3], M[3][3] = {}, Q[3][3];
      const double scale = std::ldexp(1.0, (int)(r() % 40) - 30);
      for (int i = 0; i < 3; i++) l[i] = scale * (1.0 + 9.0 * (r() / 4294967296.0));
      for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) Q[i][j] = nd(r);
      for (int j = 0; j < 3; j++) {  // Gram-Schmidt on the columns
        for (int p = 0; p < j; p++) {
          double d = 0;
          for (int i = 0; i < 3; i++) d += Q[i][j] * Q[i][p];
          for (int i = 0; i < 3; i++) Q[i][j] -= d * Q[i][p];
        }
        double s = 0;
        for (int i = 0; i < 3; i++) s += Q[i][j] * Q[i][j];
        for (int i = 0; i < 3; i++) Q[i][j] /= std::sqrt(s);
      }
      for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++)
          for (int p = 0; p < 3; p++) M[i][j] += Q[i][p] * l[p] * Q[j][p];
      float a[6] = {(float)M[0][0], (float)M[0][1], (float)M[0][2], (float)M[1][1], (float)M[1][2], (float)M[2][2]};
      const double A[3][3] = {{a[0], a[1], a[2]}, {a[1], a[3], a[4]}, {a[2], a[4], a[5]}};
      const double d64 = A[0][0] * (A[1][1] * A[2][2] - A[1][2] * A[2][1]) -
                         A[0][1] * (A[1][0] * A[2][2] - A[1][2] * A[2][0]) +
                         A[0][2] * (A[1][0] * A[2][1] - A[1][1] * A[2][0]);
      const double lmax = std::max({l[0], l[1], l[2]});
      worst_det = std::max(worst_det, std::fabs(determinant(a) - d64) / (lmax * lmax * lmax));
      float m[6];
      inverse(a, m);
      const double Mi[3][3] = {{m[0], m[1], m[2]}, {m[1], m[3], m[4]}, {m[2], m[4], m[5]}};
      for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
          double s = 0;
          for (int p = 0; p < 3; p++) s += A[i][p] * Mi[p][j];
          worst_inv = std::max(worst_inv, std::fabs(s - (i == j)));
        }
    }
    const double eps = std::numeric_limits<float>::epsilon();
    std::printf("3x3: worst |det - det64| / lmax^3 = %.3g eps, worst |A inv(A) - I| = %.3g eps\n", worst_det / eps,
                worst_inv / eps);
    CHECK(worst_det <= 8 * eps, "determinant bound");
    CHECK(worst_inv <= 64 * 10 * eps, "inverse bound");
    // singular: Inf / NaN, no trap
    const float z[6] = {0, 0, 0, 0, 0, 0};
    float m[6];
    inverse(z, m);
    CHECK(std::isnan(m[0]) && !improves(determinant(z) / 0.f, FLT_MAX) && improves(determinant(z), FLT_MAX),
          "singular matrix");
    CHECK(std::isnan(mahalanobis2(m, 1.f, 0.f, 0.f)), "NaN form");
  }
  if (failures == 0) std::printf("all mcd-rule checks passed\n");
  return failures == 0 ? 0 : 1;
}
