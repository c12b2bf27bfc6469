// Host test of the feature-distance rule (cilantro_b200/csrc/feature_rule.hpp), driven by tests/test_feature_rule.py.
//   1. with CB_NANOFLANN: rule::feature_d2 gives the bits of nanoflann's own L2_Adaptor::evalMetric (the reference's
//      vendored header) for D = 3, 6 and 9, on random and adversarial inputs;
//   2. feature_d2 >= contract_d2(xyz part) on >= 10^6 random and adversarial inputs (huge weights, subnormals, +-0,
//      tails that dominate): the claim that keeps every lower bound of the grid search valid;
//   3. rotate_tail (R (w n)) is within a few ulps of float64.
// Compile with -ffp-contract=off.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "feature_rule.hpp"

#ifdef CB_NANOFLANN
#include <nanoflann.hpp>
template <int D>
struct One {
  const float* p;
  size_t kdtree_get_point_count() const { return 1; }
  float kdtree_get_pt(size_t, size_t dim) const { return p[dim]; }
  template <class B>
  bool kdtree_get_bbox(B&) const { return false; }
};
template <int D>
float nanoflann_d2(const float* q, const float* p) {
  One<D> data{p};
  return nanoflann::L2_Adaptor<float, One<D>, float, size_t>(data).evalMetric(q, 0, D);
}
#endif

struct Rot {
  float r[9];
  float t[3];
};

static uint32_t bits(float x) {
  uint32_t b;
  std::memcpy(&b, &x, 4);
  return b;
}

template <int NT>
static float rule_d2(const float* q, const float* p) {
  const float xyz = cb::rule::contract_d2(q[0], q[1], q[2], p[0], p[1], p[2]);
  return cb::rule::feature_d2<NT>(xyz, q + 3, p + 3);
}

static float draw(std::mt19937_64& g, int mode) {
  std::uniform_real_distribution<float> u(-1.f, 1.f);
  static const float specials[] = {0.f, -0.f, 1e-40f, -1e-40f, 1.4e-45f, 1e30f, -1e30f, 3e38f, 1e-20f, 1.f};
  switch (mode) {
    case 0: return u(g);                                      // unit scale
    case 1: return u(g) * 1e30f;                              // huge weights
    case 2: return u(g) * 1e-38f;                             // subnormal differences
    case 3: return specials[g() % 10];                        // signed zeros, subnormals, extremes
    default: return u(g) * std::ldexp(1.f, (int)(g() % 200) - 100);  // mixed exponents
  }
}

int main(int argc, char** argv) {
  // argv[1] (optional): also write every sample as 21 floats (q[9], p[9], the rule's d2 for D = 3, 6, 9), so that the
  // Python side can check them against the reference's evalMetric in oracle/_ref
  std::vector<float> dump;
  std::mt19937_64 g(12345);
  int fails = 0;
  long checked_bits = 0, checked_mono = 0;
  for (long it = 0; it < 400000; ++it) {
    float q[9], p[9];
    const int mx = (int)(g() % 5), mt = (int)(g() % 5);
    for (int k = 0; k < 3; k++) {
      q[k] = draw(g, mx);
      p[k] = draw(g, mx);
    }
    for (int k = 3; k < 9; k++) {  // tails on their own scale: they may dominate or vanish
      q[k] = draw(g, mt);
      p[k] = draw(g, mt);
    }
    const float xyz = cb::rule::contract_d2(q[0], q[1], q[2], p[0], p[1], p[2]);
    const float d[3] = {xyz, rule_d2<1>(q, p), rule_d2<2>(q, p)};
    if (argc > 1) {
      dump.insert(dump.end(), q, q + 9);
      dump.insert(dump.end(), p, p + 9);
      dump.insert(dump.end(), d, d + 3);
    }
    for (int v = 0; v < 3; v++) {
      ++checked_mono;
      if (!(d[v] >= xyz) && !std::isnan(d[v]) && !std::isnan(xyz)) {
        if (fails++ < 10) printf("FAIL monotone: D=%d feature %g < xyz %g\n", 3 + 3 * v, d[v], xyz);
      }
      if (std::isnan(xyz) && !std::isnan(d[v])) {
        if (fails++ < 10) printf("FAIL NaN xyz part lost at D=%d\n", 3 + 3 * v);
      }
    }
#ifdef CB_NANOFLANN
    const float n[3] = {nanoflann_d2<3>(q, p), nanoflann_d2<6>(q, p), nanoflann_d2<9>(q, p)};
    for (int v = 0; v < 3; v++) {
      ++checked_bits;
      const bool same = bits(n[v]) == bits(d[v]) || (std::isnan(n[v]) && std::isnan(d[v]));
      if (!same && fails++ < 10) printf("FAIL bits: D=%d nanoflann %a rule %a\n", 3 + 3 * v, n[v], d[v]);
    }
#endif
  }
  // 3. rotated weighted normals against float64
  double worst = 0;
  for (int it = 0; it < 200000; ++it) {
    std::normal_distribution<double> nd;
    double a = nd(g), b = nd(g), c = nd(g), w = nd(g), qn = std::sqrt(a * a + b * b + c * c + w * w);
    a /= qn, b /= qn, c /= qn, w /= qn;
    const double R[9] = {1 - 2 * (b * b + c * c), 2 * (a * b - c * w), 2 * (a * c + b * w),
                         2 * (a * b + c * w), 1 - 2 * (a * a + c * c), 2 * (b * c - a * w),
                         2 * (a * c - b * w), 2 * (b * c + a * w), 1 - 2 * (a * a + b * b)};
    Rot T;
    for (int k = 0; k < 9; k++) T.r[k] = (float)R[k];
    const float wn = (float)std::ldexp(1.0, (int)(g() % 20) - 10);
    float v[3];
    for (int k = 0; k < 3; k++) v[k] = cb::rule::mul_rn(wn, (float)nd(g));
    float o[3];
    cb::rule::rotate_tail(T, v[0], v[1], v[2], o[0], o[1], o[2]);
    const double nv = std::sqrt((double)v[0] * v[0] + (double)v[1] * v[1] + (double)v[2] * v[2]);
    for (int r = 0; r < 3; r++) {
      const double exact = (double)T.r[3 * r] * v[0] + (double)T.r[3 * r + 1] * v[1] + (double)T.r[3 * r + 2] * v[2];
      const double e = std::fabs(o[r] - exact) / (nv * 5.960464477539063e-08);  // in ulps of |w n| (2^-24)
      worst = e > worst ? e : worst;
    }
  }
  if (worst > 6.0 && fails++ < 10) printf("FAIL rotate_tail: %.2f ulps of |w n| from float64\n", worst);
  printf("bit checks against nanoflann: %ld, monotonicity checks: %ld, rotate_tail worst %.2f ulps of |w n|\n",
         checked_bits, checked_mono, worst);
  if (argc > 1) {
    FILE* f = std::fopen(argv[1], "wb");
    if (!f || std::fwrite(dump.data(), sizeof(float), dump.size(), f) != dump.size()) return 1;
    std::fclose(f);
  }
  if (fails) return 1;
  printf("all feature-rule checks passed\n");
  return 0;
}
