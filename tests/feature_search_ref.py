"""Test helper, NOT product code: the radius-bounded feature 1-NN (feature_rule.hpp's distance, lowest index on exact
ties) restated so that it scales to 10^6 points, bit for bit the answer of the brute-force oracle
(oracle/feature_icp_oracle.cpp, feature_icp.knn1).

Candidates come from a float64 kd-tree over the packed features (fp32 inputs are exact in float64). Every fp32 rounding
of feature_d2 acts on a non-negative term, so the fp32 value f of a point with exact distance e has
|f - e| <= (D + 2) 2^-24 e, up to absolute errors of ~2^-149 per operation where terms underflow. With e_min the exact
nearest distance of a query, every point whose f can reach the fp32 minimum therefore has e <= e_min (1 + 2^-12) +
1e-30, and every other point has a strictly larger f. Those candidates are evaluated in fp32 in evalMetric's order,
one rounding per operation (numpy float32 ufuncs, no contraction), strict d2 < max_d2, ties to the lowest index.

Rows with a non-finite component are inert on either side (their distance is NaN or +inf, which never passes
d2 < max_d2 <= FLT_MAX), so they are kept out of the tree and never answer.
"""
import numpy as np
from scipy.spatial import cKDTree

REL = 2.0 ** -12
ABS = 1e-30
K = 16  # nearest candidates fetched per query; queries with more inside the band are re-queried with 4x as many


def feature_d2(q, p):
    """fp32 feature_d2 of row pairs (..., D), D = 3 / 6 / 9: ((d0² + d1²) + d2²) + d3², then (D = 6) + d4², + d5² or
    (D = 9) + g(4..7), + d8², with g(4..7) = ((d4² + d5²) + d6²) + d7²."""
    with np.errstate(over="ignore", invalid="ignore"):  # +inf and NaN distances are part of the contract
        d = np.subtract(q, p, dtype=np.float32)
        s = np.multiply(d, d, dtype=np.float32)
        D = s.shape[-1]
        acc = (s[..., 0] + s[..., 1]) + s[..., 2]
        if D == 3:
            return acc
        acc = acc + s[..., 3]
        if D == 6:
            return (acc + s[..., 4]) + s[..., 5]
        assert D == 9, D
        g = ((s[..., 4] + s[..., 5]) + s[..., 6]) + s[..., 7]
        return (acc + g) + s[..., 8]


def _nearest(tree, r, qry, q64, max_d2, ub, k):
    """fp32 minimum over each query's band, lowest tree index on ties: (best, tree index, found); recurses with a
    larger k on the queries whose band may hold more than k points."""
    n = tree.n
    k = min(k, n)
    dist, nb = tree.query(q64, k=k, distance_upper_bound=ub, workers=-1)
    dist, nb = dist.reshape(-1, k), nb.reshape(-1, k)
    found = np.isfinite(dist[:, 0])
    band = dist[:, :1] ** 2 * (1 + REL) + ABS
    inside = np.isfinite(dist) & (dist ** 2 <= band)
    cand = np.where(inside, nb, n)  # n = no candidate: a padding row of +inf
    rp = np.vstack([r, np.full((1, r.shape[1]), np.inf, np.float32)])
    order = np.argsort(cand, axis=1, kind="stable")  # by index: the first fp32 minimum is the lowest index
    cand = np.take_along_axis(cand, order, 1)
    f = feature_d2(qry[:, None, :], rp[cand])
    j = np.argmin(f, axis=1)
    rows = np.arange(qry.shape[0])
    best, bi = f[rows, j], cand[rows, j]
    more = np.flatnonzero(found & inside[:, -1]) if k < n else np.zeros(0, np.int64)
    if more.size:
        b2, i2, _ = _nearest(tree, r, qry[more], q64[more], max_d2, ub, 4 * k)
        best[more], bi[more] = b2, i2
    return best, bi, found


def knn1(ref_feats, qry_feats, max_d2, chunk=1 << 17):
    """Radius-bounded 1-NN of packed (n, D) float32 features: idx (int64, -1 = none), d2 (float32, max_d2 where none),
    the outputs of feature_icp.knn1."""
    ref = np.ascontiguousarray(ref_feats, np.float32)
    qry = np.ascontiguousarray(qry_feats, np.float32)
    max_d2 = np.float32(max_d2)
    idx = np.full(qry.shape[0], -1, np.int64)
    d2 = np.full(qry.shape[0], max_d2, np.float32)
    keep = np.flatnonzero(np.isfinite(ref).all(1))
    live = np.flatnonzero(np.isfinite(qry).all(1))
    if keep.size == 0 or live.size == 0 or not max_d2 > 0:
        return idx, d2
    r = ref[keep]
    tree = cKDTree(r.astype(np.float64))
    # no point with f < max_d2 has e >= max_d2 (1 + 2^-12)
    ub = float(np.sqrt(float(max_d2) * (1 + REL))) * (1 + 1e-9)
    for c0 in range(0, live.size, chunk):
        rows = live[c0:c0 + chunk]
        best, bi, found = _nearest(tree, r, qry[rows], qry[rows].astype(np.float64), max_d2, ub, K)
        ok = found & (best < max_d2)
        idx[rows[ok]] = keep[bi[ok]]
        d2[rows[ok]] = best[ok]
    return idx, d2


def per_query(first, second, value, n_query, by="second"):
    """A correspondence list (first = destination, second = source) read as one answer per query: for the source
    queries (by="second", the second_to_first search) or the destination queries (by="first"). Every query must appear
    at most once. Returns idx (-1 = no pair) and d2 (NaN where no pair)."""
    q, a = (second, first) if by == "second" else (first, second)
    assert np.unique(q).size == q.size, "a query appears twice in the list"
    idx = np.full(n_query, -1, np.int64)
    d2 = np.full(n_query, np.nan, np.float32)
    idx[q] = a
    d2[q] = value
    return idx, d2


def lattice_scene(n_dst, n_src, seed, h=0.125, side=(16, 16, 4), dup=0.2):
    """Exact ties everywhere: points on a dyadic lattice of spacing h (a share of them duplicated, same xyz and colour,
    another index), colours from the palette {0, h, 2h} per component, unit normals along the axes; queries on lattice
    points and cell-edge / face / cube midpoints, with palette colours and axis normals. With dyadic weights every
    feature distance is a small multiple of h^2 / 4, exact in fp32, so equal distances are equal bits."""
    rng = np.random.default_rng(seed)
    axes = np.vstack([np.eye(3), -np.eye(3)])

    def lattice(m, half):
        c = np.stack([rng.integers(0, s, m) for s in side], 1).astype(np.float64)
        if half:
            c += rng.integers(0, 2, (m, 3)) * 0.5
        return c * h

    base = n_dst - int(dup * n_dst)
    dst = lattice(base, False)
    dc = rng.integers(0, 3, (base, 3)) * h
    dn = axes[rng.integers(0, 6, base)]
    d = rng.integers(0, base, n_dst - base)
    perm = rng.permutation(n_dst)
    dst, dc, dn = (np.vstack([a, a[d]])[perm] for a in (dst, dc, dn))
    src = lattice(n_src, True)
    sc = rng.integers(0, 3, (n_src, 3)) * h
    sn = axes[rng.integers(0, 6, n_src)]
    f = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731
    return dict(dst=f(dst), dst_colors=f(dc), dst_normals=f(dn), src=f(src), src_colors=f(sc), src_normals=f(sn))
