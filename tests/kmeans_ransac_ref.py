"""A numpy restatement of what the product promises for k-means and rigid RANSAC scoring (tests only).

Not the reference's fp32 serial sums (the oracle restates those): the contracts of the device code.
  - k-means assignment: d = c - p, d2 = dx*dx + (dy*dy + dz*dz) in fp32 without FMA, j scanned ascending with a
    strict '<' from +inf (lowest j wins ties; a point whose every d2 is NaN or +inf keeps label 0).
  - Lloyd loop (cb_kmeans_cluster): float64 sums and counts over the points with three finite coordinates; the
    empty-cluster repair in ascending i from the largest count (first index on ties), the old centroid
    f32(sum) * f32(1 / count), the farthest finite member by the fp32 distance (lowest index on ties), the moved
    point leaving the sum of its cluster and not entering cluster i's; stop when no label changed (after the
    first iteration) or, with tol > 0, when the largest fp32 centroid move is < tol^2.
  - RANSAC score: q_r = (R_r0 x + (R_r1 y + R_r2 z)) + t_r, e = q - d, x = e0^2 + (e1^2 + e2^2) in fp32, inlier
    iff sqrt_rn(x) <= thresh (numpy's correctly rounded fp32 sqrt: an independent check of the device's
    precomputed x bound).
On "dyadic" inputs (multiples of 2^-10, |v| < 4) every float64 sum is exact in any order, so the device agrees
with this restatement bit for bit over whole runs.
"""
import numpy as np

import icp_ref

F32 = np.float32


def dyadic(rng, shape, lim=4.0):
    """Multiples of 2^-10 in (-lim, lim), as float32."""
    m = int(lim * 1024) - 1
    return (rng.integers(-m, m + 1, size=shape) / 1024.0).astype(F32)


def finite_rows(pts):
    return np.isfinite(np.asarray(pts, F32)).all(1)


def _d2(c, p):
    """fp32 contract distance between centroid(s) c [k, 3] and points p [n, 3] -> [n, k]."""
    c = np.asarray(c, F32)
    p = np.asarray(p, F32)
    with np.errstate(invalid="ignore", over="ignore"):
        dx = c[None, :, 0] - p[:, None, 0]
        dy = c[None, :, 1] - p[:, None, 1]
        dz = c[None, :, 2] - p[:, None, 2]
        return dx * dx + (dy * dy + dz * dz)


def kmeans_assign(pts, cent, chunk=1 << 22):
    """Labels (int64) of the strict-'<' ascending scan."""
    pts, cent = np.asarray(pts, F32).reshape(-1, 3), np.asarray(cent, F32).reshape(-1, 3)
    n, k = len(pts), len(cent)
    labels = np.zeros(n, np.int64)
    step = max(1, chunk // max(k, 1))
    for a in range(0, n, step):
        d = _d2(cent, pts[a:a + step])
        d[np.isnan(d)] = np.inf
        best = d.argmin(1)
        labels[a:a + step] = np.where(d[np.arange(len(d)), best] < np.inf, best, 0)
    return labels


def kmeans_sums(pts, labels, k):
    """float64 per-cluster sums [k, 3] and counts [k] over the finite points."""
    pts = np.asarray(pts, F32).reshape(-1, 3)
    fin = finite_rows(pts)
    s = np.zeros((k, 3))
    np.add.at(s, labels[fin], pts[fin].astype(np.float64))
    return s, np.bincount(labels[fin], minlength=k).astype(np.int64)


def kmeans_lloyd(pts, cent0, max_iter, tol):
    """cb_kmeans_cluster restated. Returns (centroids f32 [k, 3], labels int64, iterations)."""
    pts = np.asarray(pts, F32).reshape(-1, 3)
    cent = np.array(cent0, F32).reshape(-1, 3)
    k = len(cent)
    fin = finite_rows(pts)
    labels = np.zeros(len(pts), np.int64)
    tol_sq = F32(tol) * F32(tol)
    it = 0
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        while it < max_iter:
            new = kmeans_assign(pts, cent)
            changed = bool((new != labels).any())
            labels = new
            if not changed and it > 0:
                break
            old = cent.copy()
            s, cnt = kmeans_sums(pts, labels, k)
            for i in range(k):
                if cnt[i] != 0:
                    continue
                max_ind = int(np.argmax(cnt))
                inv = F32(1.0) / F32(cnt[max_ind])
                oc = s[max_ind].astype(F32) * inv
                members = np.flatnonzero((labels == max_ind) & fin)
                if len(members) == 0:
                    continue
                key = _d2(oc[None], pts[members])[:, 0].view(np.uint32)
                j = int(members[int(np.argmax(key))])
                labels[j] = i
                s[max_ind] -= pts[j].astype(np.float64)
                cnt[max_ind] -= 1
                cnt[i] += 1
            inv = F32(1.0) / cnt.astype(F32)
            cent = s.astype(F32) * inv[:, None]
            it += 1
            if tol > 0:
                mv = _d2(cent, old)[np.arange(k), np.arange(k)]
                mx = F32(0.0)
                for v in mv:  # std::max(mx, v)
                    if mx < v:
                        mx = v
                if mx < tol_sq:
                    break
    return cent, labels, it


def lloyd_cases():
    """Small dyadic Lloyd runs {name: (pts, centroids0, max_iter, tol)} at the loop's edges (n <= 1500, so the
    oracle's fp32 sums are exact too)."""
    rng = np.random.default_rng(20)
    blobs = np.vstack([dyadic(rng, (300, 3), 0.25) + c for c in ((1, 1, 1), (-2, 0, 1), (0, -2, -1))]).astype(np.float32)
    dup = np.repeat(dyadic(rng, (40, 3), 2.0), 5, axis=0)
    few = dyadic(rng, (5, 3), 2.0)
    far = dyadic(rng, (8, 3), 3.0)
    return {
        # uniform cloud, tol = 0, several iterations
        "uniform": (dyadic(rng, (1500, 3), 3.0), dyadic(rng, (24, 3), 3.0), 4, 0.0),
        # three blobs and a tol that stops the loop before the labels settle
        "tol_stop": (blobs, blobs[[0, 1, 2, 300, 600]].copy(), 50, 0.05),
        # several clusters empty in the first iteration (centroids far outside the cloud)
        "many_empty": (dyadic(rng, (800, 3), 1.0), np.vstack([dyadic(rng, (4, 3), 1.0), far + 8.0]).astype(np.float32), 3, 0.0),
        # duplicated points: farthest-member ties go to the lowest index
        "duplicates": (dup, np.vstack([dup[:3], dup[:3] + 40.0]).astype(np.float32), 3, 0.0),
        # n < K: repairs cascade, a cluster is emptied again after its turn
        "n_lt_k": (few, dyadic(rng, (9, 3), 2.0), 3, 0.0),
        "max_iter_0": (few, dyadic(rng, (3, 3), 2.0), 0, 0.0),
        "max_iter_1": (blobs, blobs[:7].copy(), 1, 0.0),
    }


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
