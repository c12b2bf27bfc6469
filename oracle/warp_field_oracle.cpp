// ORACLE (test infrastructure, NOT product code): a serial restatement of the 3-D rigid overload of
// estimateDenseWarpFieldCombinedMetric (registration/warp_field_estimation.hpp:368-715) and of the per-point update of
// CombinedMetricDenseWarpFieldICP (registration/icp_warp_field_combined_metric_dense.hpp, TransformSet::preApply,
// core/space_transformations.hpp:120-127). The ICP loop and its 1-NN search live in oracle/warp_field.py.
//
// The reference assembles the sparse At row by row and lets Eigen form At At^T; here the same rows are accumulated
// per point into the dense 6x6 data block B_i, the right-hand side g_i and, per regularisation arc, the diagonal
// coupling c = h'^2 (DESIGN §4.13 states why that is the same system). Arithmetic, selected per call:
//   Scalar = float:  blocks, vectors and the assembly in fp32, each operation rounded on its own (-ffp-contract=off),
//                    dot products accumulated in double — the device's arithmetic;
//   Scalar = double: everything in double: the reference point for tolerances.
// The CG is Eigen::ConjugateGradient with a DiagonalPreconditioner and zero initial guess, written out:
//   rhsNorm2 = |b|^2; if 0: x = 0. threshold = max(tol^2 rhsNorm2, FLT_MIN); r = b; stop if |r|^2 < threshold.
//   p = M^-1 r; absNew = r.p; loop i < maxIters: q = A p; alpha = absNew / p.q; x += alpha p; r -= alpha q;
//   break if |r|^2 < threshold; z = M^-1 r; absOld = absNew; absNew = r.z; p = z + (absNew / absOld) p; i++.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <vector>

#include "small_linalg.hpp"

#define ORC_API extern "C" __attribute__((visibility("default")))

using namespace orc;

namespace {

struct Arcs {
  std::vector<uint32_t> lo, hi;
  std::vector<float> d2;
  std::vector<std::vector<std::pair<uint32_t, uint32_t>>> inc;  // per point: (arc, other end), ascending arc
};

// arcs in the reference's equation order (:410-421, :605-617); empty lists and self-arcs give none
Arcs make_arcs(size_t n_src, const uint64_t* off, const int64_t* idx, const float* val, size_t n_reg) {
  Arcs a;
  a.inc.resize(n_src);
  for (size_t j = 0; j < n_reg; j++) {
    if (off[j + 1] - off[j] < 2) continue;
    const uint32_t c = (uint32_t)idx[off[j]];
    for (uint64_t k = off[j] + 1; k < off[j + 1]; k++) {
      const uint32_t o = (uint32_t)idx[k];
      if (o == c) continue;
      const uint32_t e = (uint32_t)a.lo.size();
      a.lo.push_back(std::min(c, o));
      a.hi.push_back(std::max(c, o));
      a.d2.push_back(val[k]);
      a.inc[c].push_back({e, o});
      a.inc[o].push_back({e, c});
    }
  }
  return a;
}

template <class S>
S sqrt_huber(S x, S delta) {  // :10-18
  const S xa = std::abs(x);
  if (xa > delta) return std::sqrt(delta * (xa - (S)0.5 * delta));
  return std::sqrt((S)0.5) * xa;
}
template <class S>
S sqrt_huber_d(S x, S delta) {  // :20-36
  const S xa = std::abs(x);
  const S v = xa > delta ? delta / ((S)2.0 * std::sqrt(delta * (xa - (S)0.5 * delta))) : std::sqrt((S)0.5);
  return x < (S)0.0 ? -v : v;
}

template <class S>
S dot3(S a0, S a1, S a2, S b0, S b1, S b2) {
  return (a0 * b0 + a1 * b1) + a2 * b2;
}

template <class S>
S trig(double (*f)(double), S x) {
  return (S)f((double)x);
}

// computeRotationTerms (:38-89): M = rot_coeffs and its derivatives, (row, col) as the reference indexes them
template <class S>
void rotation_terms(S a, S b, S c, S M[3][3], S Da[3][3], S Db[3][3], S Dc[3][3]) {
  const S sa = trig<S>(std::sin, a), ca = trig<S>(std::cos, a);
  const S sb = trig<S>(std::sin, b), cb = trig<S>(std::cos, b);
  const S sc = trig<S>(std::sin, c), cc = trig<S>(std::cos, c);
  M[0][0] = cc * cb;
  M[1][0] = -sc * ca + cc * sb * sa;
  M[2][0] = sc * sa + cc * sb * ca;
  M[0][1] = sc * cb;
  M[1][1] = cc * ca + sc * sb * sa;
  M[2][1] = -cc * sa + sc * sb * ca;
  M[0][2] = -sb;
  M[1][2] = cb * sa;
  M[2][2] = cb * ca;
  Da[0][0] = 0;
  Da[1][0] = sc * sa + cc * sb * ca;
  Da[2][0] = sc * ca - cc * sb * sa;
  Da[0][1] = 0;
  Da[1][1] = -cc * sa + sc * sb * ca;
  Da[2][1] = -cc * ca - sc * sb * sa;
  Da[0][2] = 0;
  Da[1][2] = cb * ca;
  Da[2][2] = -cb * sa;
  Db[0][0] = -cc * sb;
  Db[1][0] = cc * cb * sa;
  Db[2][0] = cc * cb * ca;
  Db[0][1] = -sc * sb;
  Db[1][1] = sc * cb * sa;
  Db[2][1] = sc * cb * ca;
  Db[0][2] = -cb;
  Db[1][2] = -sb * sa;
  Db[2][2] = -sb * ca;
  Dc[0][0] = -sc * cb;
  Dc[1][0] = -cc * ca - sc * sb * sa;
  Dc[2][0] = cc * sa - sc * sb * ca;
  Dc[0][1] = cc * cb;
  Dc[1][1] = -sc * ca + cc * sb * sa;
  Dc[2][1] = sc * sa + cc * sb * ca;
  Dc[0][2] = 0;
  Dc[1][2] = 0;
  Dc[2][2] = 0;
}

struct Prm {
  float w_pt, w_pl, stiffness, huber, reg_coeff, gn_tol, cg_tol;
  uint64_t max_gn_iter, max_cg_iter;
};

template <class S>
struct System {
  size_t n;
  std::vector<S> B, g, diag, c;  // B [n][21] upper, g [n][6], diag [n][6] of At At^T, c [arcs][6]
};

inline int upper_index(int r, int c) { return r * 6 - (r * (r - 1)) / 2 + (c - r); }

// per point: the slots of its correspondences in list order
struct CorrCsr {
  std::vector<uint32_t> off;
  std::vector<uint32_t> dst;
};
CorrCsr corr_csr(size_t n, size_t m, const uint64_t* first, const uint64_t* second) {
  CorrCsr c;
  c.off.assign(n + 1, 0);
  c.dst.resize(m);
  for (size_t k = 0; k < m; k++) c.off[second[k] + 1]++;
  for (size_t i = 0; i < n; i++) c.off[i + 1] += c.off[i];
  std::vector<uint32_t> fill(c.off.begin(), c.off.end() - 1);
  for (size_t k = 0; k < m; k++) c.dst[fill[second[k]]++] = (uint32_t)first[k];
  return c;
}

template <class S>
void assemble(const float* dst_p, const float* dst_n, const float* src_p, const CorrCsr& corr, const Arcs& arcs,
              const Prm& p, bool use_pt, bool use_pl, const std::vector<S>& x, System<S>& sys) {
  const size_t n = corr.off.size() - 1;
  sys.n = n;
  sys.B.assign(21 * n, (S)0);
  sys.g.assign(6 * n, (S)0);
  sys.diag.assign(6 * n, (S)0);
  sys.c.assign(6 * arcs.lo.size(), (S)0);
  const S w_pt = (S)std::sqrt((S)p.w_pt), w_pl = (S)std::sqrt((S)p.w_pl), w_reg = (S)std::sqrt((S)p.stiffness);
  for (size_t i = 0; i < n; i++) {
    S* B = &sys.B[21 * i];
    S* g = &sys.g[6 * i];
    const S* xi = &x[6 * i];
    auto add_row = [&](const S J[6], S res) {
      int k = 0;
      for (int r = 0; r < 6; r++) {
        for (int c = r; c < 6; c++, k++) B[k] = B[k] + J[r] * J[c];
        g[r] = g[r] + J[r] * res;
      }
    };
    for (uint32_t k = corr.off[i]; k < corr.off[i + 1] && (use_pt || use_pl); k++) {
      const size_t j = corr.dst[k];
      S M[3][3], Da[3][3], Db[3][3], Dc[3][3];
      rotation_terms<S>(xi[0], xi[1], xi[2], M, Da, Db, Dc);
      const S s[3] = {(S)src_p[3 * i], (S)src_p[3 * i + 1], (S)src_p[3 * i + 2]};
      const S d[3] = {(S)dst_p[3 * j], (S)dst_p[3 * j + 1], (S)dst_p[3 * j + 2]};
      S ts[3], das[3], dbs[3], dcs[3];
      for (int r = 0; r < 3; r++) {
        ts[r] = d[r] - (dot3<S>(M[0][r], M[1][r], M[2][r], s[0], s[1], s[2]) + xi[3 + r]);
        das[r] = dot3<S>(Da[0][r], Da[1][r], Da[2][r], s[0], s[1], s[2]);
        dbs[r] = dot3<S>(Db[0][r], Db[1][r], Db[2][r], s[0], s[1], s[2]);
        dcs[r] = dot3<S>(Dc[0][r], Dc[1][r], Dc[2][r], s[0], s[1], s[2]);
      }
      if (use_pt)  // :496-559
        for (int r = 0; r < 3; r++) {
          S J[6] = {das[r] * w_pt, dbs[r] * w_pt, dcs[r] * w_pt, 0, 0, 0};
          J[3 + r] = w_pt;
          add_row(J, ts[r] * w_pt);
        }
      if (use_pl) {  // :562-600
        const S nn[3] = {(S)dst_n[3 * j], (S)dst_n[3 * j + 1], (S)dst_n[3 * j + 2]};
        const S J[6] = {dot3<S>(nn[0], nn[1], nn[2], das[0], das[1], das[2]) * w_pl,
                        dot3<S>(nn[0], nn[1], nn[2], dbs[0], dbs[1], dbs[2]) * w_pl,
                        dot3<S>(nn[0], nn[1], nn[2], dcs[0], dcs[1], dcs[2]) * w_pl,
                        nn[0] * w_pl, nn[1] * w_pl, nn[2] * w_pl};
        add_row(J, dot3<S>(nn[0], nn[1], nn[2], ts[0], ts[1], ts[2]) * w_pl);
      }
    }
    S* dg = &sys.diag[6 * i];
    for (int u = 0; u < 6; u++) dg[u] = B[upper_index(u, u)];
    for (const auto& ie : arcs.inc[i]) {  // :603-673
      const uint32_t e = ie.first, o = ie.second;
      const bool lo = i < o;
      const S w = w_reg * (S)std::sqrt((S)std::exp((double)((S)p.reg_coeff * (S)arcs.d2[e])));
      for (int u = 0; u < 6; u++) {
        const S diff = lo ? xi[u] - x[6 * o + u] : x[6 * o + u] - xi[u];
        const S h = w * sqrt_huber_d<S>(diff, (S)p.huber);
        const S res = -(w * sqrt_huber<S>(diff, (S)p.huber));
        const S c = h * h;
        dg[u] = dg[u] + c;
        g[u] = g[u] + (lo ? h : -h) * res;
        if (lo) sys.c[6 * e + u] = c;
      }
    }
  }
}

template <class S>
void matvec(const System<S>& sys, const Arcs& arcs, const std::vector<S>& p, std::vector<S>& q) {
  for (size_t i = 0; i < sys.n; i++) {
    const S* B = &sys.B[21 * i];
    for (int r = 0; r < 6; r++) {
      S s = 0;
      for (int c = 0; c < 6; c++) s = s + B[r <= c ? upper_index(r, c) : upper_index(c, r)] * p[6 * i + c];
      q[6 * i + r] = s;
    }
    for (const auto& ie : arcs.inc[i])
      for (int u = 0; u < 6; u++)
        q[6 * i + u] = q[6 * i + u] + sys.c[6 * ie.first + u] * (p[6 * i + u] - p[6 * (size_t)ie.second + u]);
  }
}

template <class S>
double dotd(const std::vector<S>& a, const std::vector<S>& b) {
  double s = 0;
  for (size_t k = 0; k < a.size(); k++) s += (double)a[k] * (double)b[k];
  return s;
}

template <class S>
uint64_t cg(const System<S>& sys, const Arcs& arcs, uint64_t max_iter, double tol, std::vector<S>& x, float* err) {
  const size_t m = 6 * sys.n;
  x.assign(m, (S)0);
  std::vector<S> r(sys.g), p(m), q(m), z(m), inv(m);
  for (size_t k = 0; k < m; k++) inv[k] = sys.diag[k] != (S)0 ? (S)1 / sys.diag[k] : (S)1;
  const double rhs2 = dotd(r, r);
  *err = 0.f;
  if (rhs2 == 0.0) return 0;
  const double threshold = std::max(tol * tol * rhs2, (double)FLT_MIN);
  double rr = rhs2;
  uint64_t it = 0;
  if (!(rr < threshold)) {
    for (size_t k = 0; k < m; k++) p[k] = inv[k] * r[k];
    double abs_new = dotd(r, p);
    while (it < max_iter) {
      matvec(sys, arcs, p, q);
      const S alpha = (S)(abs_new / dotd(p, q));
      for (size_t k = 0; k < m; k++) {
        x[k] = x[k] + alpha * p[k];
        r[k] = r[k] - alpha * q[k];
      }
      rr = dotd(r, r);
      if (rr < threshold) break;
      for (size_t k = 0; k < m; k++) z[k] = inv[k] * r[k];
      const double abs_old = abs_new;
      abs_new = dotd(r, z);
      const S beta = (S)(abs_new / abs_old);
      for (size_t k = 0; k < m; k++) p[k] = z[k] + beta * p[k];
      it++;
    }
  }
  *err = (float)std::sqrt(rr / rhs2);
  return it;
}

// :701-712: rotation() of AngleAxis(c, Z) AngleAxis(b, Y) AngleAxis(a, X), translation (tx, ty, tz)
void unknowns_to_transform(const double* x, float* T) {
  const double ca = std::cos(x[0]), sa = std::sin(x[0]), cb = std::cos(x[1]), sb = std::sin(x[1]);
  const double cc = std::cos(x[2]), sc = std::sin(x[2]);
  M3 A;
  A.a[0][0] = cc * cb;
  A.a[0][1] = cc * sb * sa - sc * ca;
  A.a[0][2] = cc * sb * ca + sc * sa;
  A.a[1][0] = sc * cb;
  A.a[1][1] = sc * sb * sa + cc * ca;
  A.a[1][2] = sc * sb * ca - cc * sa;
  A.a[2][0] = -sb;
  A.a[2][1] = cb * sa;
  A.a[2][2] = cb * ca;
  const M3 R = nearest_rotation_col0_rule(A);
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) T[4 * r + c] = (float)R.a[r][c];
    T[4 * r + 3] = (float)x[3 + r];
  }
}

template <class S>
int solve(size_t n_dst, const float* dst_p, const float* dst_n, size_t n_src, const float* src_p, size_t n_corr,
          const uint64_t* first, const uint64_t* second, const Arcs& arcs, const Prm& p, float* T_out, float* x_out,
          uint64_t* stats, float* cg_err) {
  (void)n_dst;
  const bool use_pt = n_corr > 0 && p.w_pt > 0.f, use_pl = n_corr > 0 && p.w_pl > 0.f;
  std::vector<S> x(6 * n_src, (S)0), delta;
  bool converged = false;
  uint64_t steps = 0, cg_total = 0, cg_last = 0;
  *cg_err = 0.f;
  if (use_pt || use_pl) {  // :398-408
    const CorrCsr corr = corr_csr(n_src, n_corr, first, second);
    System<S> sys;
    const S tol2 = (S)p.gn_tol * (S)p.gn_tol;
    for (uint64_t it = 0; it < p.max_gn_iter; it++) {
      assemble<S>(dst_p, dst_n, src_p, corr, arcs, p, use_pt, use_pl, x, sys);
      cg_last = cg<S>(sys, arcs, p.max_cg_iter, (double)p.cg_tol, delta, cg_err);
      cg_total += cg_last;
      steps++;
      S mx = 0;
      for (size_t i = 0; i < n_src; i++) {
        S sq = 0;
        for (int u = 0; u < 6; u++) {
          x[6 * i + u] = x[6 * i + u] + delta[6 * i + u];
          sq = sq + delta[6 * i + u] * delta[6 * i + u];
        }
        if (sq > mx) mx = sq;
      }
      if (mx < tol2) {
        converged = true;
        break;
      }
    }
  }
  for (size_t i = 0; i < n_src; i++) {
    double xd[6];
    for (int u = 0; u < 6; u++) xd[u] = (double)(float)x[6 * i + u];
    unknowns_to_transform(xd, T_out + 12 * i);
    if (x_out)
      for (int u = 0; u < 6; u++) x_out[6 * i + u] = (float)x[6 * i + u];
  }
  stats[0] = converged;
  stats[1] = steps;
  stats[2] = cg_total;
  stats[3] = cg_last;
  return converged;
}

}  // namespace

// estimateDenseWarpFieldCombinedMetric on the (already transformed) source points: T_out [n_src][12]; stats =
// {converged, Gauss-Newton steps, CG iterations in total, CG iterations of the last step}; x_out [n_src][6] (may be
// NULL) = the unknowns, rounded to float.
ORC_API int orc_warp_solve(size_t n_dst, const float* dst_p, const float* dst_n, size_t n_src, const float* src_p,
                           size_t n_corr, const uint64_t* first, const uint64_t* second, const uint64_t* reg_off,
                           const int64_t* reg_idx, const float* reg_val, size_t n_reg, float w_pt, float w_pl,
                           float stiffness, float huber, float reg_coeff, uint64_t max_gn_iter, float gn_tol,
                           uint64_t max_cg_iter, float cg_tol, int use_double, float* T_out, float* x_out,
                           uint64_t* stats, float* cg_err) {
  const Arcs arcs = make_arcs(n_src, reg_off, reg_idx, reg_val, n_reg);
  const Prm p{w_pt, w_pl, stiffness, huber, reg_coeff, gn_tol, cg_tol, max_gn_iter, max_cg_iter};
  if (use_double)
    return solve<double>(n_dst, dst_p, dst_n, n_src, src_p, n_corr, first, second, arcs, p, T_out, x_out, stats, cg_err);
  return solve<float>(n_dst, dst_p, dst_n, n_src, src_p, n_corr, first, second, arcs, p, T_out, x_out, stats, cg_err);
}

// The normal equations at the unknowns x [n_src][6] (double mode): B [n_src][21] (upper triangle of the data block),
// g [n_src][6] (At b), diag [n_src][6] (of At At^T), arc_c [arcs][6]; arc_lo / arc_hi [arcs]. Returns the arc count
// (outputs may be NULL to size them).
ORC_API size_t orc_warp_system(const float* dst_p, const float* dst_n, size_t n_src, const float* src_p, size_t n_corr,
                               const uint64_t* first, const uint64_t* second, const uint64_t* reg_off,
                               const int64_t* reg_idx, const float* reg_val, size_t n_reg, float w_pt, float w_pl,
                               float stiffness, float huber, float reg_coeff, const double* x, double* B, double* g,
                               double* diag, double* arc_c, uint32_t* arc_lo, uint32_t* arc_hi) {
  const Arcs arcs = make_arcs(n_src, reg_off, reg_idx, reg_val, n_reg);
  if (!B) return arcs.lo.size();
  const Prm p{w_pt, w_pl, stiffness, huber, reg_coeff, 0.f, 0.f, 0, 0};
  const CorrCsr corr = corr_csr(n_src, n_corr, first, second);
  std::vector<double> xv(x, x + 6 * n_src);
  System<double> sys;
  assemble<double>(dst_p, dst_n, src_p, corr, arcs, p, n_corr > 0 && w_pt > 0.f, n_corr > 0 && w_pl > 0.f, xv, sys);
  std::memcpy(B, sys.B.data(), sys.B.size() * sizeof(double));
  std::memcpy(g, sys.g.data(), sys.g.size() * sizeof(double));
  std::memcpy(diag, sys.diag.data(), sys.diag.size() * sizeof(double));
  std::memcpy(arc_c, sys.c.data(), sys.c.size() * sizeof(double));
  std::memcpy(arc_lo, arcs.lo.data(), arcs.lo.size() * sizeof(uint32_t));
  std::memcpy(arc_hi, arcs.hi.data(), arcs.hi.size() * sizeof(uint32_t));
  return arcs.lo.size();
}

// sqrtHuberLoss (which = 0) / sqrtHuberLossDerivative (which = 1) in float, and computeRotationTerms in double (the
// four 3x3 matrices row-major into out[36]) for the unit tests.
ORC_API float orc_warp_huber(float x, float delta, int which) {
  return which ? sqrt_huber_d<float>(x, delta) : sqrt_huber<float>(x, delta);
}
ORC_API void orc_warp_rotation_terms(double a, double b, double c, double* out) {
  double M[4][3][3];
  rotation_terms<double>(a, b, c, M[0], M[1], M[2], M[3]);
  std::memcpy(out, M, sizeof(M));
}

// TransformSet::preApply (space_transformations.hpp:120-127): T[i] <- rotation(dT[i] T[i]), and
// max_i |dR_i - I|_F^2 + |dt_i|^2 (icp_warp_field_combined_metric_dense.hpp updateEstimate) in float.
ORC_API float orc_warp_compose(size_t n, const float* dT, float* T) {
  float mx = 0.f;
  for (size_t i = 0; i < n; i++) {
    const float* d = dT + 12 * i;
    float* t = T + 12 * i;
    float sq = 0.f;
    for (int c = 0; c < 3; c++)
      for (int r = 0; r < 3; r++) {
        const float e = d[4 * r + c] - (r == c ? 1.f : 0.f);
        sq = sq + e * e;
      }
    sq = sq + ((d[3] * d[3] + d[7] * d[7]) + d[11] * d[11]);
    if (sq > mx) mx = sq;
    M3 L;
    double tt[3];
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) {
        double s = 0;
        for (int k = 0; k < 3; k++) s += (double)d[4 * r + k] * (double)t[4 * k + c];
        L.a[r][c] = (double)(float)s;
      }
      double s = d[4 * r + 3];
      for (int k = 0; k < 3; k++) s += (double)d[4 * r + k] * (double)t[4 * k + 3];
      tt[r] = (double)(float)s;
    }
    const M3 R = nearest_rotation_col0_rule(L);
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) t[4 * r + c] = (float)R.a[r][c];
      t[4 * r + 3] = (float)tt[r];
    }
  }
  return mx;
}
