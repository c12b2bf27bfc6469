"""The plane-RANSAC oracle (oracle/plane_ransac_oracle.cpp) against an independent numpy statement of DESIGN §4.12:
the hypothesis plane of a sample (bit for bit, with the degenerate branches), the fp32 residual, the sample
sequence and the loop's rules (early exit, strict improvement, minimum inlier count, n < 3)."""
import numpy as np
import pytest

from oracle import ransac_plane as orp

F32 = np.float32


def np_fit(sample):
    """DESIGN §4.12's closed form in numpy float64 (one rounding per operation, no FMA)."""
    s = np.asarray(sample, F32).reshape(-1, 3)
    k = s.shape[0]
    if k < 2 or not np.all(np.isfinite(s)):
        return np.full(4, np.nan, F32)
    P = s.astype(np.float64)

    def cross(a, b):
        return np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])

    def sq(v):
        return v[0] * v[0] + (v[1] * v[1] + v[2] * v[2])

    def line(u):
        if sq(u) == 0.0:
            return np.array([0.0, 0.0, 1.0])
        j = 0
        for r in (1, 2):
            if abs(u[r]) < abs(u[j]):
                j = r
        c = cross(u, np.eye(3)[j])
        return c / np.sqrt(sq(c))

    if k == 2:
        n = line(P[1] - P[0])
        m = (P[0] + P[1]) / 2.0
    else:
        a, b, e = P[1] - P[0], P[2] - P[0], P[2] - P[1]
        c = cross(a, b)
        if np.any(c != 0.0):
            n = c / np.sqrt(sq(c))
        else:
            u = a
            if sq(b) > sq(u):
                u = b
            if sq(e) > sq(u):
                u = e
            n = line(u)
        m = ((P[0] + P[1]) + P[2]) / 3.0
    d = -(n[0] * m[0] + (n[1] * m[1] + n[2] * m[2]))
    return np.array([n[0], n[1], n[2], d]).astype(F32)


def np_residuals(pts, pl):
    p = np.asarray(pts, F32)
    pl = np.asarray(pl, F32)
    with np.errstate(invalid="ignore", over="ignore"):
        return np.abs((pl[0] * p[:, 0] + (pl[1] * p[:, 1] + pl[2] * p[:, 2])) + pl[3])


def bits(a):
    return np.asarray(a, F32).view(np.uint32)


def same_bits(a, b):
    """Equal bits, with every NaN equal to every other NaN."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(bits(a)[~np.isnan(a)], bits(b)[~np.isnan(b)])


def fit_cases():
    rng = np.random.default_rng(5)
    out = [rng.normal(size=(3, 3)) * s for s in (1e-3, 1.0, 1e3) for _ in range(30)]
    out += [rng.normal(size=(3, 3)) + 100.0 for _ in range(10)]
    base = rng.normal(size=3)
    for _ in range(10):  # collinear: exact multiples of a direction with small integer coordinates
        d = rng.integers(-3, 4, 3).astype(np.float64)
        out.append(np.array([base, base + d, base + 2 * d]))
        out.append(np.array([base + 2 * d, base, base + d]))
    out.append(np.array([[1.0, 2.0, 3.0]] * 3))                          # coincident
    out.append(np.array([[0.0, 0.0, 0.0], [0.0, 0.0, 0.0], [1.0, 0.0, 0.0]]))  # two coincident
    out.append(np.array([[1.0, 1.0, 1.0], [2.0, 2.0, 2.0], [3.0, 3.0, 3.0]]))  # ties in |u_k|
    out.append(np.array([[0.0, 0.0, 0.0], [0.0, 5.0, 0.0], [0.0, -5.0, 0.0]]))  # ties in the longest vector
    for bad in (np.nan, np.inf, -np.inf):
        s = rng.normal(size=(3, 3))
        s[1, 2] = bad
        out.append(s)
    out += [rng.normal(size=(2, 3)), np.array([[1.0, 2.0, 3.0]] * 2), np.array([[0.0, 0.0, 0.0], [0.0, 0.0, 4.0]]),
            rng.normal(size=(1, 3)), np.zeros((0, 3))]
    return out


def test_fit_bits_equal_numpy():
    for s in fit_cases():
        s = np.asarray(s, F32)
        got, want = orp.fit(s), np_fit(s)
        assert same_bits(got, want), (s, got, want)
        if s.shape[0] >= 2 and np.all(np.isfinite(s)):
            assert abs(np.linalg.norm(got[:3].astype(np.float64)) - 1.0) < 1e-6
            # every sample point lies on the plane (up to the rounding of n and d to float)
            r = np.abs(s.astype(np.float64) @ got[:3].astype(np.float64) + float(got[3]))
            assert r.max() <= 1e-5 * (1.0 + np.abs(s).max()), (s, got, r)


@pytest.mark.parametrize("thresh", [0.0, 1e-30, 0.01, np.inf, -1.0, np.nan])
def test_residual_bits_and_inliers_equal_numpy(thresh):
    rng = np.random.default_rng(2)
    pts = rng.normal(size=(3000, 3)).astype(F32)
    pts[::7, 2] = 0.0
    pts[5] = [np.nan, 0, 0]
    pts[6] = [np.inf, 1, 1]
    pts[7] = [-np.inf, 1, 1]
    pl = np.array([0.0, 0.0, 1.0, 0.0], F32)
    for plane in (pl, np_fit(pts[10:13]), np.full(4, np.nan, F32)):
        res, inl = orp.residuals(pts, plane, thresh)
        want = np_residuals(pts, plane)
        assert same_bits(res, want)
        assert np.array_equal(inl, np.nonzero(want <= F32(thresh))[0])
        assert np.array_equal(orp.score(pts, plane[None], thresh), [inl.size])


@pytest.mark.parametrize("n", [3, 4, 17, 1000])
def test_sample_sequence_is_the_rigid_estimators(orc, n):
    pts = np.random.default_rng(n).normal(size=(n, 3)).astype(F32)
    samples, planes = orp.hypotheses(pts, seed=9, iters=50)
    assert np.array_equal(samples, orc.ransac_samples(n, 3, 50, 9))
    for s, pl in zip(samples, planes):
        assert same_bits(pl, np_fit(pts[s]))


def np_loop(pts, seed, max_iter, thresh, target, samples_fn):
    """ransac_base.hpp:64-114 in numpy, without re-estimation."""
    n = pts.shape[0]
    ss = min(3, n)
    target = min(target, n)
    samples = samples_fn(n, ss, max_iter, seed) if max_iter else np.zeros((0, ss), np.int64)
    best, best_cnt, best_it, it = np.full(4, np.nan, F32), 0, 0, 0
    while it < max_iter:
        pl = np_fit(pts[samples[it]]) if ss else np.full(4, np.nan, F32)
        cnt = int((np_residuals(pts, pl) <= F32(thresh)).sum())
        it += 1
        if cnt < ss:
            continue
        if cnt > best_cnt:
            best, best_cnt, best_it = pl, cnt, it - 1
        if best_cnt >= target:
            break
    return best, best_cnt, best_it, it


@pytest.mark.parametrize("n,max_iter,target", [(0, 10, None), (1, 7, None), (2, 5, None), (3, 5, None), (50, 40, None),
                                               (50, 0, None), (50, 30, 0), (50, 30, 10**6), (2, 5, 0), (3, 6, 10)])
def test_loop_equals_numpy(orc, n, max_iter, target):
    rng = np.random.default_rng(40 + n)
    pts = np.concatenate([np.column_stack([rng.uniform(0, 1, (n, 2)), rng.normal(0, 0.001, n)])]).astype(F32)
    pts[n // 2:] = rng.uniform(0, 1, (n - n // 2, 3))
    tgt = (n // 2 + n % 2) if target is None else target
    want = np_loop(pts, 4, max_iter, 0.01, tgt, orc.ransac_samples)
    got = orp.ransac_plane(pts, 4, max_iter=max_iter, thresh=0.01, inlier_count_thresh=tgt, re_estimate=False)
    assert same_bits(got["hyp_plane"], want[0]) and same_bits(got["plane"], want[0])
    assert (got["iterations"], got["best_iteration"]) == (want[3], want[2])
    assert got["num_inliers"] == (want[1] if not np.isnan(want[0][0]) else 0)
    if n == 0:
        assert got["iterations"] == min(1, max_iter)


def test_reestimation_is_the_pca_plane_of_the_inliers():
    rng = np.random.default_rng(8)
    pts = np.column_stack([rng.uniform(0, 2, 500), rng.uniform(0, 2, 500), rng.normal(0, 0.003, 500)]).astype(F32)
    pts[300:] = rng.uniform(0, 2, (200, 3))
    got = orp.ransac_plane(pts, 1, max_iter=50, thresh=0.01, inlier_count_thresh=250)
    hyp = orp.ransac_plane(pts, 1, max_iter=50, thresh=0.01, inlier_count_thresh=250, re_estimate=False)
    _, inl = orp.residuals(pts, hyp["plane"], 0.01)
    for acc in (False, True):
        pl = orp.pca_plane(pts, inl, accum_double=acc)
        q = pts[inl].astype(np.float64)
        w, V = np.linalg.eigh(np.cov(q.T))
        assert abs(abs(float(V[:, 0] @ pl[:3])) - 1.0) < 1e-6
        assert abs(float(pl[:3] @ q.mean(0) + pl[3])) < 1e-5
    assert same_bits(got["plane"], orp.pca_plane(pts, inl))
