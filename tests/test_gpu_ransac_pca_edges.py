"""GPU rigid RANSAC and covariance / PCA at their edges.

cb_ransac_score against the numpy restatement (kmeans_ransac_ref.py) exactly: hypothesis counts on both sides of the
256-hypothesis shared-memory chunk and the 16384-hypothesis launch, pair counts at the tile and warp edges, and
thresholds where the host's x_max rewrite of sqrt_rn(x) <= thresh could slip (denormals, overflowing squares, +inf,
-0, negative, NaN). cb_ransac_rigid against the oracle's sequential loop across its 1024-hypothesis rounds and on
degenerate and non-finite samples, and its re-estimation against a float64 Kabsch. cb_mean_cov / cb_pca against
numpy float64 on the same fp32 points, around the pivot taken from the first 4096 points."""
import numpy as np
import pytest

import kmeans_ransac_ref as kr
from cilantro_b200 import synth

pytestmark = pytest.mark.gpu


# ---- cb_ransac_score ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [0, 1, 255, 256, 257, 16384, 16385])
def test_score_counts_equal_restatement(cb, ctx, H):
    T_h = kr.ransac_edge_hypotheses(H, seed=H)
    for n in (1, 31, 1023, 1024, 1025):
        dst, src = kr.ransac_edge_pairs(n, seed=n)
        d, s = cb.Cloud(ctx, dst), cb.Cloud(ctx, src)
        want = kr.ransac_counts(dst, src, T_h, kr.THRESHOLDS)
        for t, w in zip(kr.THRESHOLDS, want):
            got = cb.ransac_score(ctx, d, s, T_h, t)
            assert got.shape == (H,) and np.array_equal(got, w), (n, t, int(np.abs(got.astype(int) - w).max()))


def test_score_denormal_squares_are_not_flushed(cb, ctx):
    """Residuals near 1e-20 have squares below FLT_MIN: with flush-to-zero every one would count at any threshold."""
    rng = np.random.default_rng(4)
    src = np.zeros((2000, 3), np.float32)
    dst = np.zeros((2000, 3), np.float32)
    dst[:, 0] = (rng.uniform(0.2, 2.0, 2000) * 1e-20).astype(np.float32)
    T = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)[None]
    x = kr.ransac_x(dst, src, T)[0]
    assert (x > 0).all() and (x < np.finfo(np.float32).tiny).all()
    for t in (1e-20, 5e-21, 1.5e-20, 1e-21):
        want = kr.ransac_counts(dst, src, T, [t])[0]
        assert 0 < want[0] < 2000 or t == 1e-21
        assert np.array_equal(cb.ransac_score(ctx, cb.Cloud(ctx, dst), cb.Cloud(ctx, src), T, t), want), t


# ---- cb_ransac_rigid ----------------------------------------------------------------------------------------
def _rigid_both(cb, ctx, orc, dst, src, **kw):
    got = cb.ransac_rigid(ctx, cb.Cloud(ctx, dst), cb.Cloud(ctx, src), **kw)
    want = orc.ransac_rigid(dst, src, **kw)
    assert got["iterations"] == want["iterations"]
    assert got["best_iteration"] == want["best_iteration"]
    assert abs(got["num_inliers"] - want["num_inliers"]) <= 3
    return got, want


@pytest.mark.parametrize("n", [0, 1, 2, 3])
@pytest.mark.parametrize("re_estimate", [False, True])
def test_rigid_tiny_clouds(cb, ctx, orc, n, re_estimate):
    dst, src, _, _ = synth.ransac_pairs(max(n, 1), 1.0, seed=7)
    dst, src = dst[:n], src[:n]
    for ict in (None, n + 5):
        kw = dict(seed=3, max_iter=20, thresh=0.01, re_estimate=re_estimate)
        if ict is not None:
            kw["inlier_count_thresh"] = ict
        got, want = _rigid_both(cb, ctx, orc, dst, src, **kw)
        assert got["num_inliers"] == want["num_inliers"]
        if n == 0:
            assert got["iterations"] == want["iterations"] == 1


@pytest.mark.parametrize("max_iter", [1023, 1024, 1025, 2500])
def test_rigid_rounds_without_early_exit(cb, ctx, orc, max_iter):
    dst, src, _, _ = synth.ransac_pairs(1500, 0.3, seed=8)
    got, want = _rigid_both(cb, ctx, orc, dst, src, seed=21, max_iter=max_iter, thresh=0.01,
                            inlier_count_thresh=1501, re_estimate=False)
    assert got["iterations"] == max_iter


def _exit_in_second_round(orc, dst, src, thresh, need):
    """A seed whose first hypothesis with >= need inliers (margins of 3 either way) is in 1100 .. 1999."""
    for seed in range(500):
        samples = orc.ransac_samples(len(dst), 3, 2048, seed)
        counts = orc.ransac_score(dst, src, orc.ransac_fit_samples(dst, src, samples), thresh).astype(int)
        hit = np.flatnonzero(counts >= need)
        if len(hit) and 1100 <= hit[0] < 2000 and counts[hit[0]] >= need + 3 and counts[:hit[0]].max() < need - 3:
            return seed, int(hit[0])
    raise AssertionError("no seed found")


@pytest.mark.parametrize("re_estimate", [False, True])
def test_rigid_early_exit_inside_second_round(cb, ctx, orc, re_estimate):
    dst, src, T_ref, inl = synth.ransac_pairs(3000, 0.09, seed=9)
    need = int(0.8 * inl.sum())
    seed, first = _exit_in_second_round(orc, dst, src, 0.01, need)
    got, want = _rigid_both(cb, ctx, orc, dst, src, seed=seed, max_iter=5000, thresh=0.01,
                            inlier_count_thresh=need, re_estimate=re_estimate)
    assert got["iterations"] == first + 1 and got["best_iteration"] == first


def test_rigid_reestimate_is_float64_kabsch_of_kept_hypothesis(cb, ctx):
    dst, src, T_ref, inl = synth.ransac_pairs(20000, 0.3, seed=10)
    kw = dict(seed=5, max_iter=300, thresh=0.01, inlier_count_thresh=int(0.27 * 20000))
    d, s = cb.Cloud(ctx, dst), cb.Cloud(ctx, src)
    hyp = cb.ransac_rigid(ctx, d, s, re_estimate=False, **kw)
    fin = cb.ransac_rigid(ctx, d, s, re_estimate=True, **kw)
    assert hyp["best_iteration"] == fin["best_iteration"]
    T64, idx = kr.reestimate(dst, src, hyp["T"], 0.01)
    assert len(idx) == hyp["num_inliers"]
    assert np.abs(fin["T"].astype(np.float64) - T64).max() < 1e-6
    # the final inlier set is the one of the re-estimated model
    assert np.array_equal(fin["inliers"], kr.ransac_inliers(dst, src, fin["T"], 0.01))


@pytest.mark.parametrize("shape", ["coincident", "collinear"])
def test_rigid_degenerate_samples(cb, ctx, orc, shape):
    """Every sample is degenerate (the rotation is not unique); any valid choice maps the whole cloud."""
    rng = np.random.default_rng(12)
    if shape == "coincident":
        src = np.tile(np.float32([0.3, -0.2, 0.5]), (400, 1))
    else:
        src = (np.float32([0.1, 0.2, 0.3]) + rng.random((400, 1)) * np.float32([1.0, -0.5, 0.25])).astype(np.float32)
    dst = synth.apply(synth.t_ref_default(), src).astype(np.float32)
    for re_estimate in (False, True):
        got, want = _rigid_both(cb, ctx, orc, dst, src, seed=2, max_iter=50, thresh=0.01, re_estimate=re_estimate)
        assert got["num_inliers"] == want["num_inliers"] == 400


@pytest.mark.parametrize("re_estimate", [False, True])
def test_rigid_nonfinite_rows_in_samples(cb, ctx, orc, re_estimate):
    dst, src, _, _ = synth.ransac_pairs(30, 0.7, seed=13)
    dst[[2, 9, 17]] = kr.BAD_ROWS[:3]
    src[[5, 9, 23]] = kr.BAD_ROWS[3:]
    got, want = _rigid_both(cb, ctx, orc, dst, src, seed=4, max_iter=200, thresh=0.01, inlier_count_thresh=31,
                            re_estimate=re_estimate)
    assert got["iterations"] == 200 and np.isfinite(got["T"]).all()


# ---- cb_mean_cov / cb_pca -----------------------------------------------------------------------------------
def _cloud(kind, n, rng):
    A = np.array([[3.0, 0.5, 0.2], [0.0, 1.0, 0.3], [0.0, 0.0, 0.2]])
    if kind == "aniso":
        return rng.normal(size=(n, 3)) @ A.T
    if kind == "center_1e4":
        return rng.normal(size=(n, 3)) @ A.T + [1e4, -2e4, 3e4]
    if kind == "center_1e6":
        return rng.normal(size=(n, 3)) @ A.T + [1e6, 2e6, -1e6]
    if kind == "far_pivot":  # the first 4096 points at one end of a 1000-unit line, the rest spread over it
        t = np.concatenate([rng.uniform(0, 1, 4096), rng.uniform(0, 1000, n - 4096)])
        return np.outer(t, [0.6, 0.8, 0.0]) + rng.normal(0, 0.1, (n, 3)) + [5, 5, 5]
    if kind == "planar":
        p = rng.normal(size=(n, 3)) @ A.T
        p[:, 2] = 0.0
        return p
    if kind == "linear":
        return np.outer(rng.normal(size=n), [0.25, -0.5, 1.0]) + [1, 2, 3]
    if kind == "coincident":
        return np.tile([0.3, -7.0, 1e3], (n, 1))
    if kind == "isotropic":
        return rng.normal(size=(n, 3))
    raise ValueError(kind)


PCA_CASES = [("aniso", n) for n in (2, 3, 4095, 4096, 4097, (1 << 20) + 1)] + [
    ("center_1e4", 50000), ("center_1e6", 50000), ("center_1e6", 4097), ("far_pivot", 100000), ("planar", 30000),
    ("linear", 30000), ("coincident", 5000), ("isotropic", 200000)]


@pytest.mark.parametrize("kind,n", PCA_CASES)
def test_mean_cov_and_pca_against_float64(cb, ctx, kind, n):
    rng = np.random.default_rng(n)
    pts = _cloud(kind, n, rng).astype(np.float32)
    p = pts.astype(np.float64)
    mu = p.mean(0)
    cov = (p - mu).T @ (p - mu) / (n - 1)

    def within(got, ref):
        ref = np.asarray(ref, np.float64)
        tol = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64) + 1e-12 * np.abs(ref).max()
        return bool((np.abs(np.asarray(got, np.float64) - ref) <= tol).all())

    d = cb.Cloud(ctx, pts)
    mean, c, ok = cb.mean_cov(ctx, d)
    assert ok and within(mean, mu) and within(c, cov), (mean - mu, c - cov)
    r = cb.pca(ctx, d)
    assert r["ok"] and np.array_equal(r["mean"], mean) and np.array_equal(r["cov"], c)
    w, V = np.linalg.eigh(r["cov"].astype(np.float64))
    w, V = w[::-1], V[:, ::-1]  # descending, as the product returns them
    lmax = max(abs(w[0]), np.finfo(np.float64).tiny)
    ev = r["eigenvalues"].astype(np.float64)
    assert np.abs(ev - w).max() <= 1e-6 * lmax, (ev, w)
    E = r["eigenvectors"].astype(np.float64)
    assert np.abs(E.T @ E - np.eye(3)).max() < 1e-6 and abs(np.linalg.det(E) - 1) < 1e-6
    for j in range(3):
        gap = min(abs(w[j] - w[i]) for i in range(3) if i != j)
        if gap > 0 and 1e-6 * lmax / gap < 0.1:
            a = E[:, j] / np.linalg.norm(E[:, j])
            ang = np.arctan2(np.linalg.norm(np.cross(a, V[:, j])), abs(float(a @ V[:, j])))
            assert ang <= 1e-6 * lmax / gap, (j, ang, gap)


@pytest.mark.parametrize("row", [[np.nan] * 3, [np.inf] * 3])
@pytest.mark.parametrize("pos", [100, 4500])
def test_mean_cov_nonfinite_row(cb, ctx, row, pos):
    """Covariance semantics: a NaN point makes the mean and covariance NaN; an Inf point makes the covariance NaN
    (inf - inf) and the mean non-finite, whether or not it is among the pivot's first 4096 points."""
    pts = np.random.default_rng(14).normal(size=(5000, 3)).astype(np.float32)
    pts[pos] = row
    mean, cov, ok = cb.mean_cov(ctx, cb.Cloud(ctx, pts))
    assert ok and not np.isfinite(mean).any() and np.isnan(cov).all()
    if np.isnan(row[0]):
        assert np.isnan(mean).all()
