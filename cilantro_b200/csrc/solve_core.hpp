// Product O(1) linear algebra (double precision), compiled for the HOST and for the DEVICE: the solves the
// reference performs with Eigen once per ICP iteration. The device-resident ICP loop (icp_loop.cu) runs them
// in the last warp of the iteration's kernel, so that the iterations can be enqueued back to back without a
// host round trip; the host loop (engine modes, inner Gauss-Newton iterations, cb_solve_*) calls the same code.
//   3x3 SVD              one-sided (Hestenes) Jacobi       <- Eigen::JacobiSVD
//                                                             (registration/transform_estimation.hpp:36-44,
//                                                              core/space_transformations.hpp:43-51)
//   6x6 symmetric solve  Gaussian elimination, partial pivoting <- AtA.ldlt().solve(Atb) (:346)
//   3x3 symmetric eigen  via the SVD of the PSD covariance  <- Eigen::SelfAdjointEigenSolver
//                                                             (core/principal_component_analysis.hpp:77)
#pragma once
#include <cmath>

#if defined(__CUDACC__)
#define CB_HD __host__ __device__ __forceinline__
#else
#define CB_HD inline
#endif

namespace cb {
namespace la {

struct Mat3 {
  double m[3][3];
  CB_HD static Mat3 identity() {
    Mat3 r{};
    r.m[0][0] = r.m[1][1] = r.m[2][2] = 1.0;
    return r;
  }
};

CB_HD Mat3 mul(const Mat3& a, const Mat3& b) {
  Mat3 r{};
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) r.m[i][j] = a.m[i][0] * b.m[0][j] + a.m[i][1] * b.m[1][j] + a.m[i][2] * b.m[2][j];
  return r;
}

CB_HD Mat3 transpose(const Mat3& a) {
  Mat3 r{};
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) r.m[i][j] = a.m[j][i];
  return r;
}

CB_HD double det(const Mat3& a) {
  return a.m[0][0] * (a.m[1][1] * a.m[2][2] - a.m[1][2] * a.m[2][1]) -
         a.m[0][1] * (a.m[1][0] * a.m[2][2] - a.m[1][2] * a.m[2][0]) +
         a.m[0][2] * (a.m[1][0] * a.m[2][1] - a.m[1][1] * a.m[2][0]);
}

// A = U diag(sv) V^T, sv descending. U's columns belonging to (numerically) zero singular values
// are completed to a right- or left-handed frame as needed by the callers below, which only use
// u0, u1 and u0 x u1.
struct Svd {
  Mat3 U, V;
  double sv[3];
};

CB_HD Svd svd_hestenes(const Mat3& A) {
  double G[3][3], V[3][3];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      G[i][j] = A.m[i][j];
      V[i][j] = (i == j) ? 1.0 : 0.0;
    }
  for (int sweep = 0; sweep < 60; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        double alpha = 0, beta = 0, gamma = 0;
        for (int i = 0; i < 3; i++) {
          alpha += G[i][p] * G[i][p];
          beta += G[i][q] * G[i][q];
          gamma += G[i][p] * G[i][q];
        }
        if (gamma == 0.0 || fabs(gamma) <= 1e-17 * sqrt(alpha * beta)) continue;
        rotated = true;
        const double zeta = (beta - alpha) / (2.0 * gamma);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
        for (int i = 0; i < 3; i++) {
          const double gp = G[i][p], gq = G[i][q];
          G[i][p] = c * gp - s * gq;
          G[i][q] = s * gp + c * gq;
          const double vp = V[i][p], vq = V[i][q];
          V[i][p] = c * vp - s * vq;
          V[i][q] = s * vp + c * vq;
        }
      }
    if (!rotated) break;
  }
  double nrm[3];
  for (int j = 0; j < 3; j++) nrm[j] = sqrt(G[0][j] * G[0][j] + G[1][j] * G[1][j] + G[2][j] * G[2][j]);
  // stable descending order of three values (insertion sort as compare-exchanges). Columns are picked with selects,
  // not indexed by the order: an array indexed at run time lives in local memory on the device.
  int o0 = 0, o1 = 1, o2 = 2;
  auto nrm_of = [&](int s) { return s == 0 ? nrm[0] : (s == 1 ? nrm[1] : nrm[2]); };
  auto cmpx = [&](int& hi, int& lo) {
    if (nrm_of(lo) > nrm_of(hi)) {
      const int t = hi;
      hi = lo;
      lo = t;
    }
  };
  cmpx(o0, o1);
  cmpx(o1, o2);
  cmpx(o0, o1);  // (a no-op when the step before did not exchange)
  Svd r;
  for (int j = 0; j < 3; j++) {
    const int s = j == 0 ? o0 : (j == 1 ? o1 : o2);
    const double ns = nrm_of(s);
    r.sv[j] = ns;
    for (int i = 0; i < 3; i++) {
      const double g = s == 0 ? G[i][0] : (s == 1 ? G[i][1] : G[i][2]);
      r.V.m[i][j] = s == 0 ? V[i][0] : (s == 1 ? V[i][1] : V[i][2]);
      r.U.m[i][j] = (ns > 0.0) ? g / ns : 0.0;
    }
  }
  // complete U where singular values vanish (rank-deficient input)
  const double tiny = 1e-14 * (r.sv[0] > 1e-300 ? r.sv[0] : 1e-300);
  if (r.sv[0] <= 0.0) {
    r.U = Mat3::identity();
  } else {
    if (r.sv[1] <= tiny) {  // pick any unit vector orthogonal to u0
      int k = 0;
      double d = r.U.m[0][0];
      for (int i = 1; i < 3; i++)
        if (fabs(r.U.m[i][0]) < fabs(d)) {
          k = i;
          d = r.U.m[i][0];
        }
      const double e[3] = {k == 0 ? 1.0 : 0.0, k == 1 ? 1.0 : 0.0, k == 2 ? 1.0 : 0.0};
      double v[3] = {e[0] - d * r.U.m[0][0], e[1] - d * r.U.m[1][0], e[2] - d * r.U.m[2][0]};
      double n = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
      for (int i = 0; i < 3; i++) r.U.m[i][1] = v[i] / n;
    }
    if (r.sv[2] <= tiny) {  // u2 = u0 x u1 (sign irrelevant to the callers)
      r.U.m[0][2] = r.U.m[1][0] * r.U.m[2][1] - r.U.m[2][0] * r.U.m[1][1];
      r.U.m[1][2] = r.U.m[2][0] * r.U.m[0][1] - r.U.m[0][0] * r.U.m[2][1];
      r.U.m[2][2] = r.U.m[0][0] * r.U.m[1][1] - r.U.m[1][0] * r.U.m[0][1];
    }
  }
  return r;
}

// U V^T with the reflection repaired by negating column `flip_col` of U when det(U V) < 0:
// flip_col = 2 is the Kabsch rule (transform_estimation.hpp:38-41), flip_col = 0 is
// LinearTransform::rotation() (space_transformations.hpp:45-48).
CB_HD Mat3 rotation_from_svd(const Svd& s, int flip_col) {
  Mat3 U = s.U;
  if (det(U) * det(s.V) < 0.0)
    for (int i = 0; i < 3; i++) U.m[i][flip_col] = -U.m[i][flip_col];
  return mul(U, transpose(s.V));
}

// Orthogonal polar factor Q = U V^T of A = U S V^T by Newton's iteration X <- (mu X + X^-T / mu) / 2 (Frobenius
// scaling in the first steps), for the common case det(A) > 0 and A not close to singular: then Q is a proper
// rotation and equals what both SVD-based rules of rotation_from_svd() return (no reflection to repair), at a
// fraction of the serial latency of a Jacobi SVD (one division per step instead of several divisions and square
// roots per plane rotation) - it runs in the single-thread epilogue of every device-resident ICP iteration.
// Returns false (Q untouched) when A has det <= 0 or sigma_2 sigma_3 / sigma_1^2 < ~1e-6: the callers then take
// the SVD path, which also owns the reflection and rank-deficient rules.
CB_HD bool polar_rotation(const Mat3& A, Mat3& Q) {
  double f2 = 0;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) f2 += A.m[i][j] * A.m[i][j];
  if (!(f2 > 0.0) || !(f2 < 1e300)) return false;
  const double d0 = det(A);
  if (!(d0 > 1e-6 * f2 * sqrt(f2))) return false;
  Mat3 X = A;
  for (int k = 0; k < 40; ++k) {
    // cofactor matrix C (X^-T = C / det X)
    Mat3 C;
    C.m[0][0] = X.m[1][1] * X.m[2][2] - X.m[1][2] * X.m[2][1];
    C.m[0][1] = X.m[1][2] * X.m[2][0] - X.m[1][0] * X.m[2][2];
    C.m[0][2] = X.m[1][0] * X.m[2][1] - X.m[1][1] * X.m[2][0];
    C.m[1][0] = X.m[0][2] * X.m[2][1] - X.m[0][1] * X.m[2][2];
    C.m[1][1] = X.m[0][0] * X.m[2][2] - X.m[0][2] * X.m[2][0];
    C.m[1][2] = X.m[0][1] * X.m[2][0] - X.m[0][0] * X.m[2][1];
    C.m[2][0] = X.m[0][1] * X.m[1][2] - X.m[0][2] * X.m[1][1];
    C.m[2][1] = X.m[0][2] * X.m[1][0] - X.m[0][0] * X.m[1][2];
    C.m[2][2] = X.m[0][0] * X.m[1][1] - X.m[0][1] * X.m[1][0];
    const double dx = X.m[0][0] * C.m[0][0] + X.m[0][1] * C.m[0][1] + X.m[0][2] * C.m[0][2];
    if (!(dx > 0.0)) return false;
    const double rdx = 1.0 / dx;  // the only double-precision division of a step
    double a = 0.5, b = 0.5 * rdx;  // X <- a X + b C
    if (k < 2) {
      // Frobenius scaling mu = (|X^-T|_F / |X|_F)^(1/2) speeds up the first steps when A is far from orthogonal.
      // Any positive mu gives a valid step (the unscaled steps k >= 2 decide the limit), so single precision is
      // enough: mu^4 = |C|^2 / (det^2 |X|^2)
      double fx = 0, fc = 0;
      for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
          fx += X.m[i][j] * X.m[i][j];
          fc += C.m[i][j] * C.m[i][j];
        }
      const float mu4 = (float)(fc * rdx * rdx) / (float)fx;
      if (mu4 > 1e-30f && mu4 < 1e30f) {
        const float mu = sqrtf(sqrtf(mu4));
        a = 0.5 * (double)mu;
        b = 0.5 * rdx * (double)(1.0f / mu);
      }
    }
    double diff = 0;
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) {
        const double xn = a * X.m[i][j] + b * C.m[i][j];
        const double e = xn - X.m[i][j];
        diff += e * e;
        X.m[i][j] = xn;
      }
    if (k >= 2 && diff < 1e-28) {  // quadratic convergence: a step of 1e-14 leaves an error of ~1e-28
      Q = X;
      return true;
    }
  }
  return false;
}

// U V^T of A with the reflection rule of rotation_from_svd(.., flip_col): the polar iteration when it applies,
// else the Jacobi SVD.
CB_HD Mat3 nearest_rotation(const Mat3& A, int flip_col) {
  Mat3 Q;
  if (polar_rotation(A, Q)) return Q;
  return rotation_from_svd(svd_hestenes(A), flip_col);
}

// Solve the 6x6 system A x = b (A symmetric, given full row-major). Returns false when singular
// to working precision (x is then the least-damaged elimination result, like a failed LDLT).
CB_HD bool solve6(const double* A_in, const double* b_in, double* x) {
  const int n = 6;
  double M[6][7];
  for (int i = 0; i < n; i++) {
    for (int j = 0; j < n; j++) M[i][j] = A_in[i * n + j];
    M[i][n] = b_in[i];
  }
  bool ok = true;
  double rp[6];  // reciprocal pivots (one division per column; the back substitution re-uses them)
  for (int k = 0; k < n; k++) {
    int piv = k;
    for (int i = k + 1; i < n; i++)
      if (fabs(M[i][k]) > fabs(M[piv][k])) piv = i;
    if (piv != k)
      for (int j = 0; j <= n; j++) {
        const double t = M[k][j];
        M[k][j] = M[piv][j];
        M[piv][j] = t;
      }
    const double d = M[k][k];
    if (d == 0.0 || !(d == d)) {
      ok = false;
      rp[k] = 0.0;
      continue;
    }
    rp[k] = 1.0 / d;
    for (int i = k + 1; i < n; i++) {
      const double f = M[i][k] * rp[k];
      if (f == 0.0) continue;
      for (int j = k; j <= n; j++) M[i][j] -= f * M[k][j];
    }
  }
  for (int i = n - 1; i >= 0; i--) {
    double s = M[i][n];
    for (int j = i + 1; j < n; j++) s -= M[i][j] * x[j];
    x[i] = s * rp[i];
  }
  return ok;
}

}  // namespace la

// ---- the per-iteration solves (shared by host_solve.cpp and the device loop) -------------------------------
namespace sc {

CB_HD void t34_identity(float* T) {
  for (int i = 0; i < 12; i++) T[i] = 0.f;
  T[0] = T[5] = T[10] = 1.f;
}

// estimateTransformPointToPointMetric from reduced moments (transform_estimation.hpp:25-47). The moments are
// taken about the pivots (pd, pq) — s = {n, sum (d - pd), sum (q - pq), sum (d - pd)(q - pq)^T} — so that
// clouds far from the origin do not cancel in sigma = (sum d' q'^T)/n - mu_d' mu_q'^T (pivots of zero give the
// raw-moment form):  R = U V^T (reflection: last column of U), t = (pd + mu_d') - R (pq + mu_q').
CB_HD bool kabsch_from_moments(const double* s, const float* pd, const float* pq, float* T) {
  const double n = s[0];
  if (!(n > 0.0)) {  // :20-23
    t34_identity(T);
    return false;
  }
  const double inv_n = 1.0 / n;
  double mud[3], muq[3];
  for (int r = 0; r < 3; r++) {
    mud[r] = s[1 + r] * inv_n;
    muq[r] = s[4 + r] * inv_n;
  }
  la::Mat3 sigma;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) sigma.m[r][c] = s[7 + r * 3 + c] * inv_n - mud[r] * muq[c];
  const la::Mat3 R = la::nearest_rotation(sigma, 2);
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) T[r * 4 + c] = (float)R.m[r][c];
  for (int r = 0; r < 3; r++) {
    double t = mud[r] + (pd ? (double)pd[r] : 0.0);
    for (int c = 0; c < 3; c++) t -= (double)T[r * 4 + c] * (muq[c] + (pq ? (double)pq[c] : 0.0));
    T[r * 4 + 3] = (float)t;
  }
  return n >= 3.0;  // :47
}

// One Gauss-Newton update (transform_estimation.hpp:346-357):
//   d_theta = AtA^-1 Atb ; theta = atan(|w|) ; Ra = AngleAxis(theta, w/|w|) ; ta = cos(theta) v
//   T_out = Ra * Translation(ta) * Ra * T_in
// d_theta = AtA^-1 Atb from the reduced normal equations s28 = {n, upper AtA (21), Atb (6)}
CB_HD bool gauss_newton_solve(const double* s28, double* x) {
  double A[36], b[6];
  int k = 1;
  for (int r = 0; r < 6; r++)
    for (int c = r; c < 6; c++) {
      A[r * 6 + c] = s28[k];
      A[c * 6 + r] = s28[k];
      ++k;
    }
  for (int r = 0; r < 6; r++) b[r] = s28[22 + r];
  return la::solve6(A, b, x);
}

// the update from d_theta (already solved): T_out = Ra * Translation(ta) * Ra * T_in
CB_HD void gauss_newton_apply(const double* x, const float* Tin, float* Tout, float* dtheta_norm) {
  float dth[6];
  for (int i = 0; i < 6; i++) dth[i] = (float)x[i];  // the reference holds d_theta in fp32
  const double na = sqrt((double)dth[0] * dth[0] + (double)dth[1] * dth[1] + (double)dth[2] * dth[2]);
  const double theta = atan(na);
  double ax[3] = {0, 0, 0};
  if (na > 0.0) {
    const double rna = 1.0 / na;
    for (int i = 0; i < 3; i++) ax[i] = dth[i] * rna;
  }
  const double c = cos(theta), sn = sin(theta), k1 = 1.0 - c;
  la::Mat3 Ra;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) Ra.m[i][j] = k1 * ax[i] * ax[j] + (i == j ? c : 0.0);
  Ra.m[0][1] -= sn * ax[2];
  Ra.m[0][2] += sn * ax[1];
  Ra.m[1][0] += sn * ax[2];
  Ra.m[1][2] -= sn * ax[0];
  Ra.m[2][0] -= sn * ax[1];
  Ra.m[2][1] += sn * ax[0];
  la::Mat3 L;
  double t0[3];
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) L.m[i][j] = Tin[i * 4 + j];
    t0[i] = Tin[i * 4 + 3];
  }
  const la::Mat3 RR = la::mul(Ra, Ra);
  const la::Mat3 Lo = la::mul(RR, L);
  double t1[3], t2[3];
  for (int i = 0; i < 3; i++)
    t1[i] = Ra.m[i][0] * t0[0] + Ra.m[i][1] * t0[1] + Ra.m[i][2] * t0[2] + c * (double)dth[3 + i];
  for (int i = 0; i < 3; i++) t2[i] = Ra.m[i][0] * t1[0] + Ra.m[i][1] * t1[1] + Ra.m[i][2] * t1[2];
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) Tout[i * 4 + j] = (float)Lo.m[i][j];
    Tout[i * 4 + 3] = (float)t2[i];
  }
  double nn = 0;
  for (int i = 0; i < 6; i++) nn += (double)dth[i] * dth[i];
  if (dtheta_norm) *dtheta_norm = (float)sqrt(nn);
}

CB_HD bool gauss_newton_update(const double* s28, const float* Tin, float* Tout, float* dtheta_norm) {
  double x[6];
  const bool ok = gauss_newton_solve(s28, x);
  gauss_newton_apply(x, Tin, Tout, dtheta_norm);
  return ok;
}

// tform = Translation(dst_mean) * tform * Translation(-src_mean)   (transform_estimation.hpp:361/365)
CB_HD void uncenter(float* T, const float* dst_mean, const float* src_mean) {
  for (int i = 0; i < 3; i++) {
    double t = T[i * 4 + 3];
    for (int k = 0; k < 3; k++) t -= (double)T[i * 4 + k] * (double)src_mean[k];
    T[i * 4 + 3] = (float)(t + (double)dst_mean[i]);
  }
}

// LinearTransform::rotation() (core/space_transformations.hpp:43-51) on T's linear part
CB_HD void reorthonormalize(float* T) {
  la::Mat3 A;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) A.m[i][j] = T[i * 4 + j];
  const la::Mat3 R = la::nearest_rotation(A, 0);
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) T[i * 4 + j] = (float)R.m[i][j];
}

// out = A * B (out may alias either)
CB_HD void compose(const float* A, const float* B, float* out) {
  float r[12];
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) {
      double s = 0;
      for (int k = 0; k < 3; k++) s += (double)A[i * 4 + k] * (double)B[k * 4 + j];
      r[i * 4 + j] = (float)s;
    }
    double s = A[i * 4 + 3];
    for (int k = 0; k < 3; k++) s += (double)A[i * 4 + k] * (double)B[k * 4 + 3];
    r[i * 4 + 3] = (float)s;
  }
  for (int i = 0; i < 12; i++) out[i] = r[i];
}

// sqrt(|R - I|_F^2 + |t|^2)   (icp_single_transform_combined_metric.hpp:214-216)
CB_HD float update_norm(const float* T) {
  float dn = 0.f;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) {
      const float e = T[r * 4 + c] - (r == c ? 1.f : 0.f);
      dn += e * e;
    }
    dn += T[r * 4 + 3] * T[r * 4 + 3];
  }
  return sqrtf(dn);
}

// q = R p + t in the contract order of the query transform (DESIGN.md §2)
CB_HD void apply_point(const float* T, const float* p, float* q) {
#if defined(__CUDA_ARCH__)
  for (int r = 0; r < 3; r++)
    q[r] = __fadd_rn(__fadd_rn(__fmul_rn(T[r * 4], p[0]), __fadd_rn(__fmul_rn(T[r * 4 + 1], p[1]), __fmul_rn(T[r * 4 + 2], p[2]))),
                     T[r * 4 + 3]);
#else
  for (int r = 0; r < 3; r++) q[r] = (T[r * 4] * p[0] + (T[r * 4 + 1] * p[1] + T[r * 4 + 2] * p[2])) + T[r * 4 + 3];
#endif
}

}  // namespace sc
}  // namespace cb
