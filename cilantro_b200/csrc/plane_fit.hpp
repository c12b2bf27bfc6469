// The hypothesis plane of a RANSAC sample (DESIGN §4.12), as ONE function that compiles for the device
// (plane_fit_kernel in ransac_plane.cu) and for the host (tests/cuda/plane_fit_harness.cu checks that both builds
// give the same bits).
//
// The reference fits a sample with an fp32 PCA whose smallest eigenvector is the normal
// (model_estimation/ransac_hyperplane_estimator.hpp:103-110). For three points that eigenvector is exactly the
// normal of the plane through them; the closed form below computes it in double with every operation rounded on
// its own (no FMA), so that the result does not depend on an eigen-solver:
//   a = p1 - p0, b = p2 - p0, c = a x b;
//   c != 0: n = c / sqrt(c0^2 + (c1^2 + c2^2));
//   c == 0 (collinear or coincident): u = the longest of a, b, p2 - p1 (first on ties); u == 0: n = (0, 0, 1);
//          otherwise n = normalize(u x e_k), k = the index of the smallest |u_k| (lowest on ties);
//   m = ((p0 + p1) + p2) / 3, d = -(n0 m0 + (n1 m1 + n2 m2)); n and d rounded to float.
// A 2-point sample takes the degenerate branch with u = p1 - p0 and m = (p0 + p1) / 2. Fewer than two points, or
// a non-finite coordinate, give a NaN plane (such a plane has no inliers).
#pragma once
#if defined(__CUDACC__)
#define CB_FIT_HD __host__ __device__ __forceinline__
#else
#define CB_FIT_HD inline
#endif
#if !defined(__CUDA_ARCH__)
#include <cmath>
#endif

namespace cb {
namespace plane {

#if defined(__CUDA_ARCH__)
CB_FIT_HD double add(double a, double b) { return __dadd_rn(a, b); }
CB_FIT_HD double sub(double a, double b) { return __dsub_rn(a, b); }
CB_FIT_HD double mul(double a, double b) { return __dmul_rn(a, b); }
CB_FIT_HD double div(double a, double b) { return __ddiv_rn(a, b); }
CB_FIT_HD double sqrt_(double a) { return __dsqrt_rn(a); }
CB_FIT_HD bool finite(float x) { return isfinite(x); }
#else
// host twins: volatile operands keep the compiler from contracting or reordering
inline double add(double a, double b) { volatile double x = a, y = b; volatile double r = x + y; return r; }
inline double sub(double a, double b) { volatile double x = a, y = b; volatile double r = x - y; return r; }
inline double mul(double a, double b) { volatile double x = a, y = b; volatile double r = x * y; return r; }
inline double div(double a, double b) { volatile double x = a, y = b; volatile double r = x / y; return r; }
inline double sqrt_(double a) { volatile double x = a; return std::sqrt((double)x); }
inline bool finite(float x) { return std::isfinite(x); }
#endif

CB_FIT_HD void cross(const double* a, const double* b, double* c) {
  c[0] = sub(mul(a[1], b[2]), mul(a[2], b[1]));
  c[1] = sub(mul(a[2], b[0]), mul(a[0], b[2]));
  c[2] = sub(mul(a[0], b[1]), mul(a[1], b[0]));
}

CB_FIT_HD double norm2(const double* v) { return add(mul(v[0], v[0]), add(mul(v[1], v[1]), mul(v[2], v[2]))); }

CB_FIT_HD void scale_to_unit(const double* v, double* n) {
  const double s = sqrt_(norm2(v));
  for (int r = 0; r < 3; r++) n[r] = div(v[r], s);
}

// normal of a plane through the line along u (u != 0): normalize(u x e_k), |u_k| smallest
CB_FIT_HD void normal_of_line(const double* u, double* n) {
  int k = 0;
  for (int r = 1; r < 3; r++)
    if (fabs(u[r]) < fabs(u[k])) k = r;
  const double e[3] = {k == 0 ? 1.0 : 0.0, k == 1 ? 1.0 : 0.0, k == 2 ? 1.0 : 0.0};
  double c[3];
  cross(u, e, c);
  scale_to_unit(c, n);
}

// p: `count` points, packed xyz; out: (n0, n1, n2, d)
CB_FIT_HD void fit(const float* p, int count, float* out) {
  bool ok = count >= 2;
  for (int i = 0; i < 3 * count && i < 9; i++) ok = ok && finite(p[i]);
  if (!ok) {
    const float nan = __builtin_nanf("");
    for (int r = 0; r < 4; r++) out[r] = nan;
    return;
  }
  double P[3][3];
  for (int i = 0; i < count && i < 3; i++)
    for (int r = 0; r < 3; r++) P[i][r] = (double)p[3 * i + r];
  double n[3], m[3];
  if (count == 2) {
    double u[3];
    for (int r = 0; r < 3; r++) u[r] = sub(P[1][r], P[0][r]);
    if (norm2(u) == 0.0) {
      n[0] = 0.0; n[1] = 0.0; n[2] = 1.0;
    } else {
      normal_of_line(u, n);
    }
    for (int r = 0; r < 3; r++) m[r] = div(add(P[0][r], P[1][r]), 2.0);
  } else {
    double a[3], b[3], c[3];
    for (int r = 0; r < 3; r++) {
      a[r] = sub(P[1][r], P[0][r]);
      b[r] = sub(P[2][r], P[0][r]);
    }
    cross(a, b, c);
    if (c[0] != 0.0 || c[1] != 0.0 || c[2] != 0.0) {
      scale_to_unit(c, n);
    } else {
      double e[3];
      for (int r = 0; r < 3; r++) e[r] = sub(P[2][r], P[1][r]);
      const double* u = a;
      double lu = norm2(a);
      if (norm2(b) > lu) { u = b; lu = norm2(b); }
      if (norm2(e) > lu) { u = e; lu = norm2(e); }
      if (lu == 0.0) {
        n[0] = 0.0; n[1] = 0.0; n[2] = 1.0;
      } else {
        normal_of_line(u, n);
      }
    }
    for (int r = 0; r < 3; r++) m[r] = div(add(add(P[0][r], P[1][r]), P[2][r]), 3.0);
  }
  const double d = -add(mul(n[0], m[0]), add(mul(n[1], m[1]), mul(n[2], m[2])));
  for (int r = 0; r < 3; r++) out[r] = (float)n[r];
  out[3] = (float)d;
}

}  // namespace plane
}  // namespace cb
