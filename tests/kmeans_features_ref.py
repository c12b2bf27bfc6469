"""A numpy restatement of what the product promises for k-means (cb_kmeans_*, DESIGN §4.3 and §4.17; tests only).

The one restatement for every D: clouds are D = 3, cb_vectors sets any D >= 1. Not the reference's fp32 serial sums
(the oracle restates those): the contracts of the device code.
  - distance: d = c - p per component in fp32, then the right fold without FMA,
    acc = d[D-1]^2; acc = d[j]^2 + acc for j = D-2 .. 0 (at D = 3: dx*dx + (dy*dy + dz*dz));
  - assignment: strict '<' over ascending j from +inf (lowest j wins ties; a row whose every d2 is NaN or +inf keeps
    label 0);
  - Lloyd loop (cb_kmeans_cluster, cb_kmeans_cluster_vectors): float64 sums and counts over the rows whose D
    components are finite; the empty-cluster repair in ascending i from the largest count (first index on ties), the
    old centroid f32(sum) * f32(1 / count), the farthest finite member by the fp32 distance (lowest index on ties), the
    moved row leaving the sum of its cluster and not entering cluster i's; stop when no label changed (after the first
    iteration) or, with tol > 0, when the largest fp32 centroid move is < tol^2.
On dyadic inputs (multiples of 2^-10, |v| < 4) and n small enough, every float64 sum is exact in any order, so the
device agrees with this restatement bit for bit over whole runs.
"""
import numpy as np

from kmeans_ransac_ref import dyadic

F32 = np.float32


def d2(cent, pts):
    """fp32 contract distance [n, k] between rows pts [n, D] and centroids cent [k, D]."""
    c = np.asarray(cent, F32)
    p = np.asarray(pts, F32)
    acc = np.zeros((len(p), len(c)), F32)
    with np.errstate(invalid="ignore", over="ignore"):
        for j in range(c.shape[1] - 1, -1, -1):
            d = c[None, :, j] - p[:, None, j]
            acc = d * d + acc
    return acc


def fold_rows(a, b):
    """fp32 contract distance between matching rows of a and b [k, D] -> [k]."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    acc = np.zeros(len(a), F32)
    with np.errstate(invalid="ignore", over="ignore"):
        for j in range(a.shape[1] - 1, -1, -1):
            d = a[:, j] - b[:, j]
            acc = d * d + acc
    return acc


def assign(pts, cent, chunk=1 << 22):
    """Labels (int64) of the strict-'<' ascending scan."""
    pts, cent = np.asarray(pts, F32), np.asarray(cent, F32)
    n, k = len(pts), len(cent)
    labels = np.zeros(n, np.int64)
    step = max(1, chunk // max(k, 1))
    for a in range(0, n, step):
        d = d2(cent, pts[a:a + step])
        d[np.isnan(d)] = np.inf
        best = d.argmin(1)
        labels[a:a + step] = np.where(d[np.arange(len(d)), best] < np.inf, best, 0)
    return labels


def sums(pts, labels, k):
    """float64 per-cluster sums [k, D] and counts [k] over the finite rows."""
    pts = np.asarray(pts, F32)
    fin = np.isfinite(pts).all(1)
    s = np.zeros((k, pts.shape[1]))
    np.add.at(s, labels[fin], pts[fin].astype(np.float64))
    return s, np.bincount(labels[fin], minlength=k).astype(np.int64)


def lloyd(pts, cent0, max_iter, tol):
    """cb_kmeans_cluster / cb_kmeans_cluster_vectors restated. Returns (centroids f32 [k, D], labels int64, iterations)."""
    pts = np.asarray(pts, F32)
    cent = np.array(cent0, F32)
    k = len(cent)
    fin = np.isfinite(pts).all(1)
    labels = np.zeros(len(pts), np.int64)
    tol_sq = F32(tol) * F32(tol)
    it = 0
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        while it < max_iter:
            new = assign(pts, cent)
            changed = bool((new != labels).any())
            labels = new
            if not changed and it > 0:
                break
            old = cent.copy()
            s, cnt = sums(pts, labels, k)
            for i in range(k):
                if cnt[i] != 0:
                    continue
                max_ind = int(np.argmax(cnt))
                inv = F32(1.0) / F32(cnt[max_ind])
                oc = s[max_ind].astype(F32) * inv
                members = np.flatnonzero((labels == max_ind) & fin)
                if len(members) == 0:
                    continue
                key = d2(oc[None], pts[members])[:, 0].view(np.uint32)
                j = int(members[int(np.argmax(key))])
                labels[j] = i
                s[max_ind] -= pts[j].astype(np.float64)
                cnt[max_ind] -= 1
                cnt[i] += 1
            inv = F32(1.0) / cnt.astype(F32)
            cent = s.astype(F32) * inv[:, None]
            it += 1
            if tol > 0:
                mx = F32(0.0)
                for v in fold_rows(cent, old):  # std::max(mx, v)
                    if mx < v:
                        mx = v
                if mx < tol_sq:
                    break
    return cent, labels, it


def lloyd_cases(D, seed=0):
    """Small dyadic Lloyd runs {name: (pts, centroids0, max_iter, tol)} at the loop's edges in D dimensions."""
    rng = np.random.default_rng(seed + 31 * D)
    shifts = [np.full(D, v, F32) for v in (1.0, -2.0, 0.5)]
    blobs = np.vstack([dyadic(rng, (200, D), 0.25) + c for c in shifts]).astype(F32)
    dup = np.repeat(dyadic(rng, (30, D), 2.0), 5, axis=0)
    few = dyadic(rng, (5, D), 2.0)
    far = dyadic(rng, (6, D), 3.0)
    return {
        "uniform": (dyadic(rng, (1200, D), 3.0), dyadic(rng, (20, D), 3.0), 4, 0.0),
        "tol_stop": (blobs, blobs[[0, 1, 2, 200, 400]].copy(), 50, 0.05),
        "many_empty": (dyadic(rng, (600, D), 1.0), np.vstack([dyadic(rng, (4, D), 1.0), far + 8.0]).astype(F32), 3, 0.0),
        "duplicates": (dup, np.vstack([dup[:3], dup[:3] + 40.0]).astype(F32), 3, 0.0),
        "n_lt_k": (few, dyadic(rng, (9, D), 2.0), 3, 0.0),
        "max_iter_0": (few, dyadic(rng, (3, D), 2.0), 0, 0.0),
        "max_iter_1": (blobs, blobs[:7].copy(), 1, 0.0),
        "empty_set": (np.zeros((0, D), F32), dyadic(rng, (3, D), 2.0), 5, 0.0),
    }


def cloud_lloyd_cases():
    """Small dyadic Lloyd runs {name: (pts [n, 3], centroids0, max_iter, tol)} at the loop's edges on clouds (n <= 1500,
    so the oracle's fp32 sums are exact too)."""
    rng = np.random.default_rng(20)
    blobs = np.vstack([dyadic(rng, (300, 3), 0.25) + c for c in ((1, 1, 1), (-2, 0, 1), (0, -2, -1))]).astype(F32)
    dup = np.repeat(dyadic(rng, (40, 3), 2.0), 5, axis=0)
    few = dyadic(rng, (5, 3), 2.0)
    far = dyadic(rng, (8, 3), 3.0)
    return {
        # uniform cloud, tol = 0, several iterations
        "uniform": (dyadic(rng, (1500, 3), 3.0), dyadic(rng, (24, 3), 3.0), 4, 0.0),
        # three blobs and a tol that stops the loop before the labels settle
        "tol_stop": (blobs, blobs[[0, 1, 2, 300, 600]].copy(), 50, 0.05),
        # several clusters empty in the first iteration (centroids far outside the cloud)
        "many_empty": (dyadic(rng, (800, 3), 1.0), np.vstack([dyadic(rng, (4, 3), 1.0), far + 8.0]).astype(F32), 3, 0.0),
        # duplicated points: farthest-member ties go to the lowest index
        "duplicates": (dup, np.vstack([dup[:3], dup[:3] + 40.0]).astype(F32), 3, 0.0),
        # n < K: repairs cascade, a cluster is emptied again after its turn
        "n_lt_k": (few, dyadic(rng, (9, 3), 2.0), 3, 0.0),
        "max_iter_0": (few, dyadic(rng, (3, 3), 2.0), 0, 0.0),
        "max_iter_1": (blobs, blobs[:7].copy(), 1, 0.0),
    }
