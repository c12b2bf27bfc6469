// ORACLE — test infrastructure, NOT product code.
// Serial restatement of NormalEstimation<float, 3, MinimumCovarianceDeterminant<float, 3>> (core/normal_estimation.hpp:
// 279-421 over core/covariance.hpp:185-371) under the contract of DESIGN §4.15, built by oracle/Makefile into
// oracle/librobust_normals_oracle.so with -ffp-contract=off. It does not include the product's rule header: the draws
// come from the installed libstdc++ (std::minstd_rand0, std::uniform_int_distribution<size_t>), the kept subset from
// std::sort on (key, position) with NaN as +inf, and the 3x3 algebra is written out again here, one rounding per
// operation in the order DESIGN §4.15 states. Neighbourhoods are given (the tests take them from BruteKnn: ascending
// (d2, index)). The eigen step is the plain oracle's (double Jacobi of small_linalg.hpp, DESIGN §6: unpinned).
#include <algorithm>
#include <cmath>
#include <cfloat>
#include <cstddef>
#include <cstdint>
#include <limits>
#include <random>
#include <utility>
#include <vector>

#include "small_linalg.hpp"

#define ORC_API extern "C" __attribute__((visibility("default")))

namespace {

const float kNaN = std::numeric_limits<float>::quiet_NaN();

uint32_t fmix32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x85ebca6bu;
  x ^= x >> 13;
  x *= 0xc2b2ae35u;
  x ^= x >> 16;
  return x;
}

struct Cov {
  float mean[3];
  float c[6];  // xx, xy, xz, yy, yz, zz
};

// covariance.hpp:121-135 in fp32, points in the order given
Cov mean_cov(const float* pts, const std::vector<int64_t>& idx) {
  Cov r;
  float s[3] = {0.f, 0.f, 0.f};
  for (int64_t i : idx)
    for (int c = 0; c < 3; c++) s[c] = s[c] + pts[3 * i + c];
  const float inv = 1.0f / (float)idx.size();
  for (int c = 0; c < 3; c++) r.mean[c] = inv * s[c];
  float cs[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int64_t i : idx) {
    const float dx = pts[3 * i] - r.mean[0], dy = pts[3 * i + 1] - r.mean[1], dz = pts[3 * i + 2] - r.mean[2];
    cs[0] = cs[0] + dx * dx;
    cs[1] = cs[1] + dx * dy;
    cs[2] = cs[2] + dx * dz;
    cs[3] = cs[3] + dy * dy;
    cs[4] = cs[4] + dy * dz;
    cs[5] = cs[5] + dz * dz;
  }
  const float invm1 = 1.0f / (float)(idx.size() - 1);
  for (int c = 0; c < 6; c++) r.c[c] = invm1 * cs[c];
  return r;
}

// cofactor matrix of the symmetric a (symmetric itself), determinant by the first row
void cof(const float* a, float* c) {
  c[0] = a[3] * a[5] - a[4] * a[4];
  c[1] = a[2] * a[4] - a[1] * a[5];
  c[2] = a[1] * a[4] - a[2] * a[3];
  c[3] = a[0] * a[5] - a[2] * a[2];
  c[4] = a[1] * a[2] - a[0] * a[4];
  c[5] = a[0] * a[3] - a[1] * a[1];
}
float det(const float* a) {
  float c[6];
  cof(a, c);
  return (a[0] * c[0] + a[1] * c[1]) + a[2] * c[2];
}
void inv(const float* a, float* m) {
  float c[6];
  cof(a, c);
  const float r = 1.0f / ((a[0] * c[0] + a[1] * c[1]) + a[2] * c[2]);
  for (int i = 0; i < 6; i++) m[i] = c[i] * r;
}
float maha(const float* m, const float* p, const float* mean) {
  const float dx = p[0] - mean[0], dy = p[1] - mean[1], dz = p[2] - mean[2];
  const float r0 = (m[0] * dx + m[1] * dy) + m[2] * dz;
  const float r1 = (m[1] * dx + m[3] * dy) + m[4] * dz;
  const float r2 = (m[2] * dx + m[4] * dy) + m[5] * dz;
  return (dx * r0 + dy * r1) + dz * r2;
}

}  // namespace

// nbr: n x stride neighbour indices (search order), cnt: their counts. Outputs may be NULL: normals 3n, curvature n,
// cov6 6n, status n, kept n x stride (the winning trial's kept positions in selection order, -1 after h; the whole
// neighbourhood when the plain covariance was taken), h n.
ORC_API void orc_mcd_normals(const float* pts, size_t n, const int64_t* nbr, size_t stride, const uint32_t* cnt,
                             int num_trials, int num_refinements, float inlier_ratio, float chi2, int min_size,
                             uint32_t seed, const float* view_point3, const float* ref_normals, float* normals,
                             float* curvature, float* cov6, uint8_t* status, int32_t* kept, uint32_t* h_out) {
  const bool use_vp = view_point3 && std::isfinite(view_point3[0]) && std::isfinite(view_point3[1]) &&
                      std::isfinite(view_point3[2]);
  const size_t ms = (size_t)min_size;
#pragma omp parallel for schedule(dynamic, 64)
  for (size_t i = 0; i < n; i++) {
    const size_t m = cnt[i];
    std::vector<int64_t> nb(nbr + i * stride, nbr + i * stride + m);
    uint8_t st = 0;
    Cov best{};
    std::vector<int64_t> best_kept;
    size_t h = m;
    if (m < ms) {
      st = 1;
    } else if (m == ms) {
      best = mean_cov(pts, nb);
      best_kept = nb;
    } else {
      // h = min(max(min, llround(ratio * size)), size) (covariance.hpp:316-318); llround < 0 wraps to a huge size_t
      const long long r = std::llround(inlier_ratio * (float)m);
      const size_t hr = r < 0 ? SIZE_MAX : (size_t)r;
      h = std::min(std::max(ms, hr), m);
      if (h == m) {
        best = mean_cov(pts, nb);
        best_kept = nb;
      } else {
        std::minstd_rand0 gen(fmix32(seed ^ fmix32((uint32_t)i + 0x9e3779b9u)));
        std::uniform_int_distribution<size_t> pick(0, m - 1);
        float best_det = FLT_MAX;
        bool found = false;
        for (int t = 0; t < num_trials; t++) {
          std::vector<int64_t> sample(ms);
          for (size_t s = 0; s < ms; s++) sample[s] = nb[pick(gen)];
          Cov cur = mean_cov(pts, sample);
          std::vector<int64_t> sel;
          for (int rf = 0; rf < num_refinements; rf++) {
            float mi[6];
            inv(cur.c, mi);
            std::vector<std::pair<float, size_t>> keys(m);
            for (size_t j = 0; j < m; j++) {
              float q = maha(mi, pts + 3 * nb[j], cur.mean);
              if (std::isnan(q)) q = INFINITY;
              keys[j] = {q, j};
            }
            std::sort(keys.begin(), keys.end(), [](const std::pair<float, size_t>& a, const std::pair<float, size_t>& b) {
              return a.first < b.first || (a.first == b.first && a.second < b.second);  // -0 == +0
            });
            sel.assign(h, 0);
            for (size_t j = 0; j < h; j++) sel[j] = nb[keys[j].second];
            cur = mean_cov(pts, sel);
          }
          const float d = det(cur.c);
          if (std::isfinite(d) && d < best_det) {
            best_det = d;
            best = cur;
            best_kept = sel.empty() ? sample : sel;
            found = true;
          }
        }
        if (!found) st = 3;
      }
      if (st == 0 && chi2 > 0.f) {
        float mi[6];
        inv(best.c, mi);
        if (!(maha(mi, pts + 3 * nb[0], best.mean) <= chi2)) st = 2;
      }
    }
    if (status) status[i] = st;
    if (h_out) h_out[i] = (uint32_t)h;
    if (kept)
      for (size_t j = 0; j < stride; j++) kept[i * stride + j] = j < best_kept.size() ? (int32_t)best_kept[j] : -1;
    if (st != 0) {
      if (normals) normals[3 * i] = normals[3 * i + 1] = normals[3 * i + 2] = kNaN;
      if (curvature) curvature[i] = kNaN;
      if (cov6)
        for (int c = 0; c < 6; c++) cov6[6 * i + c] = kNaN;
      continue;
    }
    const float* cv = best.c;
    if (cov6)
      for (int c = 0; c < 6; c++) cov6[6 * i + c] = cv[c];
    orc::M3 C, V;
    C.a[0][0] = cv[0]; C.a[0][1] = C.a[1][0] = cv[1]; C.a[0][2] = C.a[2][0] = cv[2];
    C.a[1][1] = cv[3]; C.a[1][2] = C.a[2][1] = cv[4]; C.a[2][2] = cv[5];
    double w[3];
    orc::sym3_eigen(C, w, V);
    float nv[3] = {(float)V.a[0][0], (float)V.a[1][0], (float)V.a[2][0]};
    if (ref_normals) {  // normal_estimation.hpp:351-355
      const float* r = ref_normals + 3 * i;
      if (nv[0] * r[0] + (nv[1] * r[1] + nv[2] * r[2]) < 0.f)
        for (int c = 0; c < 3; c++) nv[c] = -nv[c];
    } else if (use_vp) {  // :325-329
      const float ex = view_point3[0] - pts[3 * i], ey = view_point3[1] - pts[3 * i + 1],
                  ez = view_point3[2] - pts[3 * i + 2];
      if (nv[0] * ex + (nv[1] * ey + nv[2] * ez) < 0.f)
        for (int c = 0; c < 3; c++) nv[c] = -nv[c];
    }
    if (normals)
      for (int c = 0; c < 3; c++) normals[3 * i + c] = nv[c];
    if (curvature) curvature[i] = (float)(w[0] / (w[0] + w[1] + w[2]));
  }
}
