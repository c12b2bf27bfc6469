"""GPU k-means over D-dimensional rows (capi.Vectors, cb_kmeans_*_vectors) against the numpy restatement
kmeans_features_ref.py: the assignment at the kernel's dimension-chunk (16), tile (128) and warp edges and on both sides
of the shared / global sums switch (K x (D + 1) x 8 B <= 184 KiB), ties, whole Lloyd runs through repairs, tol stops and
non-finite rows, the D = 3 path against cb_kmeans_cluster on a Cloud, non-dyadic data at scale, argument errors,
launch counts and device memory. On dyadic inputs the device's double atomics are exact in any order, so labels, sums,
centroids and iteration counts agree bit for bit."""
import ctypes as C

import numpy as np
import pytest

import kmeans_features_ref as kf
import kmeans_ransac_ref as kr
from test_gpu_device_memory import pool_used  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

DIMS = [1, 2, 4, 5, 6, 9, 16, 17, 32, 33, 128, 1024]


def _same_f32(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


def _check_assign(cb, ctx, pts, cent):
    labels, sums, counts = cb.kmeans_assign(ctx, cb.Vectors(ctx, pts), cent)
    want = kf.assign(pts, cent)
    ws, wc = kf.sums(pts, want, len(cent))
    assert np.array_equal(labels, want), (pts.shape, len(cent), int((labels != want).sum()))
    assert np.array_equal(counts, wc) and np.array_equal(sums, ws), (pts.shape, len(cent))


@pytest.mark.parametrize("D", DIMS)
def test_assign_at_tile_and_warp_edges(cb, ctx, D):
    rng = np.random.default_rng(D)
    ks = (1, 127, 128, 129, 257) if D <= 128 else (1, 129)
    ns = (1, 31, 127, 128, 129, 1000) if D <= 128 else (1, 31, 129)
    for k in ks:
        cent = kr.dyadic(rng, (k, D), 3.0)
        for n in ns:
            _check_assign(cb, ctx, kr.dyadic(rng, (n, D), 3.0), cent)


# the largest K whose K x (D + 1) double sums fit the 184 KiB block budget, and the next one
@pytest.mark.parametrize("D,k", [(6, 3364), (6, 3365), (32, 713), (32, 714), (2, 7850), (2, 7851)])
def test_assign_on_both_sides_of_the_sums_switch(cb, ctx, D, k):
    rng = np.random.default_rng(k)
    _check_assign(cb, ctx, kr.dyadic(rng, (3000, D), 3.0), kr.dyadic(rng, (k, D), 3.0))


@pytest.mark.parametrize("D", [2, 6, 17])
def test_ties_go_to_the_lowest_index(cb, ctx, D):
    rng = np.random.default_rng(40 + D)
    base = kr.dyadic(rng, (20, D), 2.0)
    cent = np.vstack([base, base[::-1], base]).astype(np.float32)  # every centroid three times
    # centroids 0 and 1 lie 0.5 either side of the last point, far from everything else
    mid = np.zeros((2, D), np.float32)
    mid[:, 0] = (49.5, 50.5)
    tie = np.zeros((1, D), np.float32)
    tie[0, 0] = 50.0
    pts = np.vstack([base, kr.dyadic(rng, (500, D), 2.0), tie]).astype(np.float32)
    labels, _, _ = cb.kmeans_assign(ctx, cb.Vectors(ctx, pts), np.vstack([mid, cent]).astype(np.float32))
    want = kf.assign(pts, np.vstack([mid, cent]))
    assert np.array_equal(labels, want)
    assert labels[-1] == 0  # equidistant from centroids 0 and 1
    assert (labels[:20] == 2 + np.arange(20)).all()  # the first of the three copies


@pytest.mark.parametrize("D", [2, 6, 17, 40])
@pytest.mark.parametrize("case", list(kf.lloyd_cases(2)))
def test_lloyd_runs_bit_identical(cb, ctx, D, case):
    pts, cent0, max_iter, tol = kf.lloyd_cases(D)[case]
    res = cb.kmeans_cluster(ctx, cb.Vectors(ctx, pts), cent0, max_iter=max_iter, tol=tol)
    rc, rl, rit = kf.lloyd(pts, cent0, max_iter, tol)
    assert res["iterations"] == rit
    assert np.array_equal(res["labels"], rl)
    assert _same_f32(res["centroids"], rc)
    if case == "tol_stop":
        assert rit < max_iter
    if case == "max_iter_0":
        assert rit == 0 and not rl.any() and _same_f32(res["centroids"], cent0)


@pytest.mark.parametrize("D", [5, 33])
def test_non_finite_rows_change_nothing_else(cb, ctx, D):
    pts, cent0, max_iter, tol = kf.lloyd_cases(D)["uniform"]
    bad = np.full((6, D), 0.5, np.float32)
    for i, v in enumerate((np.nan, np.inf, -np.inf, np.nan, np.inf, np.nan)):
        bad[i, (7 * i) % D] = v
    mixed = np.insert(pts, [0, 10, 10, 500, len(pts), len(pts)], bad, axis=0)
    good = np.isfinite(mixed).all(1)
    clean = cb.kmeans_cluster(ctx, cb.Vectors(ctx, pts), cent0, max_iter=max_iter, tol=tol)
    res = cb.kmeans_cluster(ctx, cb.Vectors(ctx, mixed), cent0, max_iter=max_iter, tol=tol)
    assert res["iterations"] == clean["iterations"]
    assert _same_f32(res["centroids"], clean["centroids"])
    assert np.array_equal(res["labels"][good], clean["labels"]) and not res["labels"][~good].any()
    rc, rl, rit = kf.lloyd(mixed, cent0, max_iter, tol)
    assert rit == res["iterations"] and np.array_equal(res["labels"], rl) and _same_f32(res["centroids"], rc)


@pytest.mark.parametrize("case", list(kf.cloud_lloyd_cases()))
def test_d3_vectors_equal_cloud(cb, ctx, case):
    pts, cent0, max_iter, tol = kf.cloud_lloyd_cases()[case]
    a = cb.kmeans_cluster(ctx, cb.Cloud(ctx, pts), cent0, max_iter=max_iter, tol=tol)
    b = cb.kmeans_cluster(ctx, cb.Vectors(ctx, pts), cent0, max_iter=max_iter, tol=tol)
    assert a["iterations"] == b["iterations"] and a["kernel_launches"] == b["kernel_launches"]
    assert np.array_equal(a["labels"], b["labels"]) and _same_f32(a["centroids"], b["centroids"])
    la, sa, ca = cb.kmeans_assign(ctx, cb.Cloud(ctx, pts), cent0)
    lb, sb, cbn = cb.kmeans_assign(ctx, cb.Vectors(ctx, pts), cent0)
    assert np.array_equal(la, lb) and np.array_equal(sa, sb) and np.array_equal(ca, cbn)


def test_non_dyadic_at_scale(cb, ctx):
    """1 M x D = 32 x K = 256, uniform floats: every assignment bit-exact; over a run, the double sums' order only moves
    centroids by a few ulps, so labels differ from the restatement's run at boundary points only."""
    rng = np.random.default_rng(9)
    pts = rng.standard_normal((1_000_000, 32)).astype(np.float32)
    cent0 = pts[rng.choice(len(pts), 256, replace=False)].copy()
    v = cb.Vectors(ctx, pts)
    labels, sums, counts = cb.kmeans_assign(ctx, v, cent0)
    want = kf.assign(pts, cent0)
    assert np.array_equal(labels, want), int((labels != want).sum())
    ws, wc = kf.sums(pts, want, 256)
    assert np.array_equal(counts, wc) and np.allclose(sums, ws, rtol=1e-12, atol=1e-9)
    res = cb.kmeans_cluster(ctx, v, cent0, max_iter=2, tol=0.0)
    rc, rl, rit = kf.lloyd(pts, cent0, 2, 0.0)
    assert res["iterations"] == rit == 2
    assert np.allclose(res["centroids"], rc, rtol=0, atol=1e-5)
    flips = int((res["labels"] != rl).sum())
    assert flips <= 100, f"{flips} label differences (boundary points only)"
    # the last assignment of the run is bit-exact against the centroids it started from
    step, _, _ = cb.kmeans_assign(ctx, v, res["centroids"])
    assert np.array_equal(step, kf.assign(pts, res["centroids"]))


def test_argument_errors(cb, ctx):
    lib = cb.lib()
    pts = np.zeros((4, 5), np.float32)
    h = C.c_void_p()
    with pytest.raises(cb.CbError):
        cb.Vectors(ctx, np.zeros((4, 0), np.float32))  # D = 0
    assert lib.cb_vectors_create(ctx.h, cb._p(pts), C.c_size_t(4), C.c_int(-2), C.byref(h)) == -1
    assert lib.cb_vectors_create(ctx.h, None, C.c_size_t(4), C.c_int(5), C.byref(h)) == -1
    assert lib.cb_vectors_create(None, cb._p(pts), C.c_size_t(4), C.c_int(5), C.byref(h)) == -1
    assert lib.cb_vectors_create(ctx.h, cb._p(pts), C.c_size_t(4), C.c_int(5), None) == -1
    v = cb.Vectors(ctx, pts)
    assert lib.cb_vectors_size(v.h) == 4 and lib.cb_vectors_size(None) == 0
    cent = np.zeros((2, 5), np.float32)
    with pytest.raises(cb.CbError):
        cb.kmeans_assign(ctx, v, np.zeros((0, 5), np.float32))  # k = 0
    with pytest.raises(cb.CbError):
        cb.kmeans_cluster(ctx, v, np.zeros((0, 5), np.float32))
    res = cb.KMeansResult()
    assert lib.cb_kmeans_cluster_vectors(ctx.h, None, cb._p(cent), C.c_size_t(2), C.c_size_t(3), C.c_float(0), None,
                                         C.byref(res)) == -1
    assert lib.cb_kmeans_cluster_vectors(ctx.h, v.h, None, C.c_size_t(2), C.c_size_t(3), C.c_float(0), None,
                                         C.byref(res)) == -1
    assert lib.cb_kmeans_assign_vectors(None, v.h, cb._p(cent), C.c_size_t(2), None, None, None) == -1
    with pytest.raises(AssertionError):
        cb.kmeans_assign(ctx, v, np.zeros((2, 4), np.float32))  # centroids of another dimension


def test_launches_per_iteration(cb, ctx):
    """One assignment kernel per loop pass, plus one farthest-member kernel per repaired cluster."""
    pts, cent0, _, _ = kf.lloyd_cases(6)["tol_stop"]
    v = cb.Vectors(ctx, pts)
    res = cb.kmeans_cluster(ctx, v, cent0, max_iter=50, tol=0.0)
    assert res["iterations"] < 50
    assert res["kernel_launches"] == res["iterations"] + 1  # the last pass finds no label changed
    pts, cent0, max_iter, _ = kf.lloyd_cases(6)["many_empty"]
    res = cb.kmeans_cluster(ctx, cb.Vectors(ctx, pts), cent0, max_iter=1, tol=0.0)
    _, cnt = kf.sums(pts, kf.assign(pts, cent0), len(cent0))
    assert res["kernel_launches"] == 1 + int((cnt == 0).sum()) > 1


def test_no_device_memory_growth(cb, ctx, pool_used):
    pts, cent0, max_iter, tol = kf.lloyd_cases(9)["many_empty"]

    def once():
        v = cb.Vectors(ctx, pts)
        cb.kmeans_cluster(ctx, v, cent0, max_iter=max_iter, tol=tol)
        cb.kmeans_assign(ctx, v, cent0)
        with pytest.raises(cb.CbError):
            cb.kmeans_assign(ctx, v, np.zeros((0, 9), np.float32))
        v.close()

    once()
    before = pool_used()
    for _ in range(5):
        once()
    assert pool_used() <= before
