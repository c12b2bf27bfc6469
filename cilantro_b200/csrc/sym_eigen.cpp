// Symmetric eigen-decomposition of a D x D matrix on the host, fp64 (product code; no device). PCA over D-dimensional
// rows (principal_component_analysis.hpp:76-84) hands it the fp32-rounded covariance. Written from Golub & Van Loan,
// "Matrix Computations" (4th ed.): Householder tridiagonalisation (Algorithm 8.3.1, with the Householder vectors of
// Algorithm 5.1.1 and the backward accumulation of Q of §5.1.6), then the symmetric QR algorithm (Algorithm 8.3.3)
// whose implicit steps with a Wilkinson shift (Algorithm 8.3.2) chase the bulge from the top of each unreduced block,
// accumulating the Givens rotations into the eigenvectors: O(D^3). Every inner loop runs along contiguous rows.
#include "cb_internal.hpp"
#include <algorithm>
#include <cmath>
#include <limits>
#include <numeric>
#include <vector>

namespace {

// Householder tridiagonalisation of the symmetric row-major n x n matrix a: on return diag / off hold T
// (off[k] couples k and k + 1) and q (row-major) the orthogonal Q with Q^T A Q = T.
void tridiagonalize(std::vector<double>& a, int n, std::vector<double>& diag, std::vector<double>& off,
                    std::vector<double>& q) {
  auto A = [&](int i, int j) -> double& { return a[(size_t)i * n + j]; };
  std::vector<double> v((size_t)n), p((size_t)n), beta((size_t)n, 0.0), vs((size_t)n * n, 0.0);
  for (int k = 0; k + 2 < n; k++) {
    // v, beta with (I - beta v v^T) x = mu e1 for x = A(k+1:n, k), v(0) = 1 (Algorithm 5.1.1)
    const int m = n - k - 1;
    const double x0 = A(k + 1, k);
    double sigma = 0.0;
    for (int i = 1; i < m; i++) sigma += A(k + 1 + i, k) * A(k + 1 + i, k);
    if (sigma == 0.0) {  // already tridiagonal in this column
      off[k] = x0;
      continue;
    }
    const double mu = std::sqrt(x0 * x0 + sigma);
    const double v0 = x0 <= 0.0 ? x0 - mu : -sigma / (x0 + mu);
    const double b = 2.0 * v0 * v0 / (sigma + v0 * v0);
    v[0] = 1.0;
    for (int i = 1; i < m; i++) v[i] = A(k + 1 + i, k) / v0;
    off[k] = mu;
    // p = b A22 v, w = p - (b p^T v / 2) v, A22 -= v w^T + w v^T (A22 = A(k+1:n, k+1:n), row by row)
    double pv = 0.0;
    for (int i = 0; i < m; i++) {
      const double* row = &A(k + 1 + i, k + 1);
      double t = 0.0;
      for (int j = 0; j < m; j++) t += row[j] * v[j];
      p[i] = b * t;
      pv += p[i] * v[i];
    }
    const double half = 0.5 * b * pv;
    for (int i = 0; i < m; i++) p[i] -= half * v[i];  // p is now w
    for (int i = 0; i < m; i++) {
      double* row = &A(k + 1 + i, k + 1);
      const double vi = v[i], wi = p[i];
      for (int j = 0; j < m; j++) row[j] -= vi * p[j] + wi * v[j];
    }
    beta[k] = b;
    std::copy(v.begin(), v.begin() + m, vs.begin() + (size_t)k * n);
  }
  for (int k = 0; k < n; k++) diag[k] = A(k, k);
  if (n >= 2) off[n - 2] = A(n - 1, n - 2);
  // Q = H_0 H_1 ... H_{n-3}, accumulated backwards: Q(k+1:n, k+1:n) = (I - beta v v^T) Q(k+1:n, k+1:n)
  std::fill(q.begin(), q.end(), 0.0);
  for (int i = 0; i < n; i++) q[(size_t)i * n + i] = 1.0;
  for (int k = n - 3; k >= 0; k--) {
    if (beta[k] == 0.0) continue;
    const int m = n - k - 1;
    const double* vk = &vs[(size_t)k * n];
    std::fill(p.begin(), p.begin() + m, 0.0);  // p = v^T Q22
    for (int i = 0; i < m; i++) {
      const double* row = &q[(size_t)(k + 1 + i) * n + k + 1];
      for (int j = 0; j < m; j++) p[j] += vk[i] * row[j];
    }
    for (int i = 0; i < m; i++) {
      double* row = &q[(size_t)(k + 1 + i) * n + k + 1];
      const double s = beta[k] * vk[i];
      for (int j = 0; j < m; j++) row[j] -= s * p[j];
    }
  }
}

// Symmetric QR on T = tridiag(diag, off) (Algorithm 8.3.3). zt holds Q transposed (row i = column i of Q), so each
// rotation combines two contiguous rows. An off-diagonal entry is set to zero once it is below
// eps (|d_k| + |d_k+1|) (the test of Algorithm 8.3.3) or below eps ||T|| (a perturbation no larger than the rounding
// the reduction already made). On return diag holds the eigenvalues and row i of zt the eigenvector of diag[i].
// false: a block did not split within 100 implicit steps.
bool symmetric_qr(std::vector<double>& diag, std::vector<double>& off, std::vector<double>& zt, int n) {
  const double eps = std::numeric_limits<double>::epsilon();
  // ||T||_inf: rounding leaves errors of about eps ||T|| in every entry, so an off-diagonal entry below that is as good
  // as zero even where its diagonal neighbours are far smaller (graded matrices, eigenvalues 1e-24 ||T|| and below)
  double tnorm = 0.0;
  for (int k = 0; k < n; k++)
    tnorm = std::max(tnorm, std::fabs(diag[k]) + (k + 1 < n ? std::fabs(off[k]) : 0.0) +
                                (k > 0 ? std::fabs(off[k - 1]) : 0.0));
  auto negligible = [&](int k) {
    return std::fabs(off[k]) <= eps * (std::fabs(diag[k]) + std::fabs(diag[k + 1])) ||
           std::fabs(off[k]) <= eps * tnorm;
  };
  int hi = n - 1, steps = 0;
  while (hi > 0) {
    if (negligible(hi - 1)) {  // the bottom eigenvalue has split off
      off[hi - 1] = 0.0;
      hi--;
      steps = 0;
      continue;
    }
    int lo = hi - 1;  // the unreduced block [lo, hi]
    while (lo > 0 && !negligible(lo - 1)) lo--;
    if (lo > 0) off[lo - 1] = 0.0;
    if (++steps > 100) return false;
    // Wilkinson shift: the eigenvalue of the trailing 2 x 2 closer to its last diagonal entry (Algorithm 8.3.2)
    const double dlt = 0.5 * (diag[hi - 1] - diag[hi]);
    const double bb = off[hi - 1];
    const double den = dlt + (dlt >= 0.0 ? 1.0 : -1.0) * std::hypot(dlt, bb);
    const double shift = diag[hi] - bb * (bb / den);
    double x = diag[lo] - shift, z = off[lo];
    for (int k = lo; k < hi; k++) {
      // the rotation R on coordinates k, k+1 with R (x, z)^T = (r, 0)^T, applied as T = R T R^T
      const double r = std::hypot(x, z);
      const double c = r > 0.0 ? x / r : 1.0, s = r > 0.0 ? z / r : 0.0;
      if (k > lo) off[k - 1] = r;
      const double ak = diag[k], ak1 = diag[k + 1], bk = off[k];
      diag[k] = c * c * ak + 2.0 * c * s * bk + s * s * ak1;
      diag[k + 1] = s * s * ak - 2.0 * c * s * bk + c * c * ak1;
      off[k] = c * s * (ak1 - ak) + (c * c - s * s) * bk;
      if (k + 1 < hi) {  // the bulge at (k, k+2) becomes the next z
        x = off[k];
        z = s * off[k + 1];
        off[k + 1] *= c;
      }
      double* zk = &zt[(size_t)k * n];
      double* zk1 = &zt[(size_t)(k + 1) * n];
      for (int i = 0; i < n; i++) {
        const double u = zk[i], w = zk1[i];
        zk[i] = c * u + s * w;
        zk1[i] = c * w - s * u;
      }
    }
  }
  return true;
}

// sign of det(M) (row-major n x n, overwritten) by Gaussian elimination with partial pivoting
int det_sign(std::vector<double>& M, int n) {
  int sign = 1;
  for (int c = 0; c < n; c++) {
    int piv = c;
    for (int r = c + 1; r < n; r++)
      if (std::fabs(M[(size_t)r * n + c]) > std::fabs(M[(size_t)piv * n + c])) piv = r;
    if (M[(size_t)piv * n + c] == 0.0) return 0;
    if (piv != c) {
      for (int k = 0; k < n; k++) std::swap(M[(size_t)piv * n + k], M[(size_t)c * n + k]);
      sign = -sign;
    }
    const double p = M[(size_t)c * n + c];
    if (p < 0.0) sign = -sign;
    for (int r = c + 1; r < n; r++) {
      const double f = M[(size_t)r * n + c] / p;
      if (f == 0.0) continue;
      for (int k = c; k < n; k++) M[(size_t)r * n + k] -= f * M[(size_t)c * n + k];
    }
  }
  return sign;
}

}  // namespace

namespace cb {

// Eigenvalues descending, eigenvectors as unit columns of evecs (row-major D x D), all fp64 and without the sign rules.
// Returns 1; 0 for a non-finite entry and -1 when the QR iteration did not converge, both with all-NaN output.
int sym_eigen_f64(const double* A, int D, double* evals, double* evecs) {
  const size_t DD = (size_t)D * D;
  double amax = 0.0;
  bool finite = true;
  for (size_t i = 0; i < DD; i++) {
    finite = finite && std::isfinite(A[i]);
    amax = std::max(amax, std::fabs(A[i]));
  }
  const double nan = std::numeric_limits<double>::quiet_NaN();
  auto fail = [&](int rc) {
    std::fill(evals, evals + D, nan);
    std::fill(evecs, evecs + DD, nan);
    return rc;
  };
  if (!finite) return fail(0);
  // work on A / max|A|: no over- or underflow in the squares whatever the scale of the input
  const double scale = amax > 0.0 ? amax : 1.0;
  std::vector<double> a(DD), d((size_t)D), e((size_t)D, 0.0), q(DD);
  for (int i = 0; i < D; i++)
    for (int j = 0; j < D; j++) a[(size_t)i * D + j] = 0.5 * (A[(size_t)i * D + j] + A[(size_t)j * D + i]) / scale;
  tridiagonalize(a, D, d, e, q);
  std::vector<double> zt(DD);
  for (int i = 0; i < D; i++)
    for (int j = 0; j < D; j++) zt[(size_t)j * D + i] = q[(size_t)i * D + j];
  if (!symmetric_qr(d, e, zt, D)) return fail(-1);
  std::vector<int> order((size_t)D);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return d[x] > d[y]; });
  for (int j = 0; j < D; j++) {
    const double* v = &zt[(size_t)order[j] * D];
    for (int i = 0; i < D; i++) evecs[(size_t)i * D + j] = v[i];
    evals[j] = d[order[j]] * scale;
  }
  return 1;
}

// sym_eigen_f64, then each eigenvector signed so that its largest-magnitude component is positive (the lowest index on
// ties), the last column negated when det < 0, and everything rounded to fp32.
int sym_eigen(const double* A, int D, float* evals, float* evecs) {
  const size_t DD = (size_t)D * D;
  std::vector<double> d((size_t)D), E(DD);
  const int rc = sym_eigen_f64(A, D, d.data(), E.data());
  if (rc != 1) {
    std::fill(evals, evals + D, std::numeric_limits<float>::quiet_NaN());
    std::fill(evecs, evecs + DD, std::numeric_limits<float>::quiet_NaN());
    return rc;
  }
  for (int j = 0; j < D; j++) {
    int big = 0;
    for (int i = 1; i < D; i++)
      if (std::fabs(E[(size_t)i * D + j]) > std::fabs(E[(size_t)big * D + j])) big = i;
    if (E[(size_t)big * D + j] < 0.0)
      for (int i = 0; i < D; i++) E[(size_t)i * D + j] = -E[(size_t)i * D + j];
  }
  std::vector<double> M(E);
  if (det_sign(M, D) < 0)
    for (int i = 0; i < D; i++) E[(size_t)i * D + D - 1] = -E[(size_t)i * D + D - 1];
  for (int j = 0; j < D; j++) evals[j] = (float)d[j];
  for (size_t i = 0; i < DD; i++) evecs[i] = (float)E[i];
  return 1;
}

}  // namespace cb

extern "C" {

int cb_solve_sym_eigen(const double* A, int D, float* evals, float* evecs) {
  CB_CHECK(A && evals && evecs && D >= 1, CB_ERR_INVALID, "bad arguments");
  const int rc = cb::sym_eigen(A, D, evals, evecs);
  CB_CHECK(rc >= 0, CB_ERR_UNSUPPORTED, "symmetric eigen-solve: the QR iteration did not converge");
  return rc;
}

}  // extern "C"
