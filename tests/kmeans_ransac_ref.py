"""A numpy restatement of what the product promises for rigid RANSAC scoring, and the inputs the k-means and RANSAC
tests share (tests only). k-means is restated once, for every D, in kmeans_features_ref.py.

Not the reference's fp32 serial sums (the oracle restates those): the contract of the device code.
  - RANSAC score: q_r = (R_r0 x + (R_r1 y + R_r2 z)) + t_r, e = q - d, x = e0^2 + (e1^2 + e2^2) in fp32, inlier
    iff sqrt_rn(x) <= thresh (numpy's correctly rounded fp32 sqrt: an independent check of the device's
    precomputed x bound).
On "dyadic" inputs (multiples of 2^-10, |v| < 4) every float64 sum is exact in any order: the device's double
atomics then agree with a float64 restatement bit for bit over whole runs.
"""
import numpy as np

import icp_ref

F32 = np.float32


def dyadic(rng, shape, lim=4.0):
    """Multiples of 2^-10 in (-lim, lim), as float32."""
    m = int(lim * 1024) - 1
    return (rng.integers(-m, m + 1, size=shape) / 1024.0).astype(F32)


def ransac_x(dst, src, T_h):
    """Squared residual x [H, n] of every pair under every hypothesis, fp32 contract order."""
    dst, src = np.asarray(dst, F32).reshape(-1, 3), np.asarray(src, F32).reshape(-1, 3)
    T = np.asarray(T_h, F32).reshape(-1, 3, 4)
    with np.errstate(invalid="ignore", over="ignore"):
        e = []
        for r in range(3):
            q = (T[:, r, 0, None] * src[None, :, 0] + (T[:, r, 1, None] * src[None, :, 1] +
                                                       T[:, r, 2, None] * src[None, :, 2])) + T[:, r, 3, None]
            e.append(q - dst[None, :, r])
        return e[0] * e[0] + (e[1] * e[1] + e[2] * e[2])


def ransac_counts(dst, src, T_h, threshs, chunk=1024):
    """uint32 counts [H] of pairs with sqrt_rn(x) <= thresh, one array per entry of threshs."""
    T = np.asarray(T_h, F32).reshape(-1, 3, 4)
    out = [np.zeros(len(T), np.uint32) for _ in threshs]
    for a in range(0, len(T), chunk):
        with np.errstate(invalid="ignore"):
            r = np.sqrt(ransac_x(dst, src, T[a:a + chunk]))
            for o, t in zip(out, threshs):
                o[a:a + chunk] = (r <= F32(t)).sum(1)
    return out


# thresholds at the edges of the x <= x_max rewrite: zero and -0, the smallest denormal, a threshold whose residuals
# have denormal squares, the largest thresholds whose square does / does not overflow, +inf, negative and NaN
THRESHOLDS = (0.0, -0.0, 1.4e-45, 1e-20, 0.01, 1.8446743e19, 3e38, np.inf, -1.0, np.nan)

BAD_ROWS = np.array([[np.nan, np.nan, np.nan], [np.inf, np.inf, np.inf], [-np.inf, -np.inf, -np.inf],
                     [np.inf, -np.inf, 0.5], [0.5, np.nan, 0.5], [-np.inf, 0.5, np.inf]], F32)


def ransac_edge_pairs(n, seed):
    """n (dst, src) pairs cycling through residual regimes, by row index mod 10: 0-3 noisy matches (residuals
    around 0.01), 4 exact matches, 5 residuals near 1e-20 (denormal squares), 6 residuals within a few ulps of
    sqrt(FLT_MAX), 7 residuals near 3e38 (x overflows), 8 a BAD_ROWS row in dst or src, 9 unrelated points."""
    rng = np.random.default_rng(seed)
    src = rng.uniform(-1, 1, (n, 3)).astype(F32)
    dst = (src + rng.normal(0, 0.01, (n, 3))).astype(F32)
    cat = np.arange(n) % 10
    dst[cat == 4] = src[cat == 4]
    for c, scale in ((5, 1e-20), (6, None), (7, 3e38)):
        m = np.flatnonzero(cat == c)
        src[m] = 0.0
        dst[m] = 0.0
        if scale is None:
            base = np.array([1.8446743e19], F32).view(np.uint32)
            dst[m, 0] = (base + rng.integers(-3, 4, len(m)).astype(np.uint32)).view(F32)
        else:
            dst[m, 0] = (rng.uniform(0.3, 1.1, len(m)) * scale).astype(F32)
            dst[m, 1] = (rng.uniform(-0.5, 0.5, len(m)) * scale).astype(F32)
    m = np.flatnonzero(cat == 8)
    for k, j in enumerate(m):
        (dst if k % 2 else src)[j] = BAD_ROWS[k % len(BAD_ROWS)]
    m = np.flatnonzero(cat == 9)
    dst[m] = rng.uniform(-1, 1, (len(m), 3)).astype(F32)
    return dst, src


def ransac_edge_hypotheses(H, seed):
    """H fp32 [R | t]: the identity, the identity shifted by 0.005 in x, then small random rotations and shifts."""
    rng = np.random.default_rng(seed)
    T = np.zeros((H, 3, 4), F32)
    for h in range(H):
        if h < 2:
            R, t = np.eye(3), np.array([0.005 * h, 0.0, 0.0])
        else:
            w = rng.normal(0, 0.01, 3)
            a = np.linalg.norm(w)
            K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) / a
            R = np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K
            t = rng.normal(0, 0.005, 3)
        T[h, :, :3] = R
        T[h, :, 3] = t
    return T


def ransac_inliers(dst, src, T, thresh):
    with np.errstate(invalid="ignore"):
        return np.flatnonzero(np.sqrt(ransac_x(dst, src, T)[0]) <= F32(thresh))


def reestimate(dst, src, T, thresh):
    """The re-estimation step: float64 Kabsch over the inliers of hypothesis T (dst <- src)."""
    idx = ransac_inliers(dst, src, T, thresh)
    Tk, _ = icp_ref.kabsch(np.asarray(dst)[idx], np.asarray(src)[idx])
    return Tk, idx
