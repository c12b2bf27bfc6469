"""numpy restatement of covariance, PCA projection and reconstruction over D-dimensional rows (DESIGN §4.18).

mean_cov is the float64 two-pass covariance of the reference (core/covariance.hpp:30-179) with its per-dimension
non-finite semantics and its sample-size expressions; the device result is within one fp32 spacing of it (plus the
bound of DESIGN §4.18). project / reconstruct are the pinned fp32 folds, one rounding per operation, bit for bit.
"""
import numpy as np


def mean_cov(rows, subset=None, min_sample_size=2):
    """(mean [D] float64, cov [D, D] float64, ok) of rows [n, D] (or of rows[subset])."""
    rows = np.asarray(rows, np.float32)
    D = rows.shape[1]
    x = rows if subset is None else rows[np.asarray(subset, np.int64)]
    n = x.shape[0]
    if n < min_sample_size:
        return np.full(D, np.nan), np.full((D, D), np.nan), False
    if n == 0:  # (1 / 0) * 0; (1 / (n - 1)) * 0 with n - 1 = -1 (Eigen::Index) or 2^64 - 1 (size_t)
        return np.full(D, np.nan), np.full((D, D), 0.0 if subset is not None else -0.0), True
    p = x.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        mean = p.sum(0) / n
        if n == 1:
            return p[0].copy(), np.full((D, D), np.nan), True
        bad = ~np.isfinite(p).all(0)
        c = np.where(bad[None, :], 0.0, p - np.where(bad, 0.0, mean)[None, :])
        cov = c.T @ c / (n - 1)
    cov[bad, :] = np.nan
    cov[:, bad] = np.nan
    return mean, cov, True


def project(rows, mean, evecs, k):
    """acc = 0; for d = 0 .. D-1: acc = acc + E[d][j] * (p_d - mean_d), fp32."""
    rows = np.asarray(rows, np.float32)
    mean = np.asarray(mean, np.float32)
    E = np.asarray(evecs, np.float32)
    c = rows - mean[None, :]
    acc = np.zeros((rows.shape[0], k), np.float32)
    for d in range(rows.shape[1]):
        acc = acc + E[d, :k][None, :] * c[:, d:d + 1]
    return acc


def reconstruct(q, mean, evecs):
    """acc = 0; for j = 0 .. k-1: acc = acc + E[r][j] * q_j; out_r = acc + mean_r, fp32."""
    q = np.asarray(q, np.float32)
    mean = np.asarray(mean, np.float32)
    E = np.asarray(evecs, np.float32)
    acc = np.zeros((q.shape[0], mean.size), np.float32)
    for j in range(q.shape[1]):
        acc = acc + E[:, j][None, :] * q[:, j:j + 1]
    return acc + mean[None, :]


def within_cov_bound(mean, cov, ref_mean, ref_cov):
    """The accuracy bound of DESIGN §4.18: each covariance entry within one fp32 spacing of the float64 value plus
    2^-30 sqrt(C_ii C_jj), each mean entry within one spacing plus 2^-30 sqrt(C_jj); non-finite entries must match the
    restatement's pattern (NaN where it is NaN, the same infinity where it is infinite)."""
    def check(got, ref, slack):
        got = np.asarray(got, np.float64)
        fin = np.isfinite(ref)
        if not np.array_equal(np.isnan(got), np.isnan(ref)):
            return False
        if not np.array_equal(got[np.isinf(ref)], ref[np.isinf(ref)]):
            return False
        r = ref[fin]
        tol = np.spacing(np.abs(r).astype(np.float32)).astype(np.float64) + slack[fin]
        return bool((np.abs(got[fin] - r) <= tol).all())

    diag = np.where(np.isfinite(np.diag(ref_cov)), np.abs(np.diag(ref_cov)), 0.0)
    cslack = 2.0 ** -30 * np.sqrt(np.outer(diag, diag))
    mslack = 2.0 ** -30 * np.sqrt(diag)
    return check(mean, ref_mean, mslack) and check(cov, ref_cov, cslack)
