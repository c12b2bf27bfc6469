"""GPU k-means against the float64 restatement (kmeans_features_ref.py) at the kernel's edges: centroid counts at the
shared-memory chunk (1024) and the shared / global sums switch (K = 5888 | 5889), point counts at the tile and warp
edges, whole Lloyd runs through repairs, ties and tol stops, and non-finite points. On dyadic inputs the device's
double atomics are exact in any order, so labels, sums, centroids and iteration counts agree bit for bit."""
import numpy as np
import pytest

import kmeans_features_ref as kf
import kmeans_ransac_ref as kr

pytestmark = pytest.mark.gpu


def _same_f32(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


@pytest.mark.parametrize("k", [1, 1023, 1024, 1025, 2048, 5888, 5889, 8192])
def test_assign_at_chunk_and_sums_path_edges(cb, ctx, k):
    rng = np.random.default_rng(k)
    cent = kr.dyadic(rng, (k, 3), 3.0)
    for n in (1, 31, 1023, 1024, 1025, 4097):
        pts = kr.dyadic(rng, (n, 3), 3.0)
        labels, sums, counts = cb.kmeans_assign(ctx, cb.Cloud(ctx, pts), cent)
        want = kf.assign(pts, cent)
        ws, wc = kf.sums(pts, want, k)
        assert np.array_equal(labels, want), (n, int((labels != want).sum()))
        assert np.array_equal(counts, wc) and np.array_equal(sums, ws), n


@pytest.mark.parametrize("k", [5889, 8192])
def test_lloyd_on_global_sums_path(cb, ctx, k):
    rng = np.random.default_rng(k + 1)
    pts = kr.dyadic(rng, (12000, 3), 3.0)
    cent0 = pts[rng.choice(len(pts), k, replace=False)].copy()
    res = cb.kmeans_cluster(ctx, cb.Cloud(ctx, pts), cent0, max_iter=3, tol=0.0)
    rc, rl, rit = kf.lloyd(pts, cent0, 3, 0.0)
    assert res["iterations"] == rit == 3
    assert np.array_equal(res["labels"], rl)
    assert _same_f32(res["centroids"], rc)


@pytest.mark.parametrize("case", list(kf.cloud_lloyd_cases()))
def test_lloyd_runs_bit_identical(cb, ctx, case):
    pts, cent0, max_iter, tol = kf.cloud_lloyd_cases()[case]
    res = cb.kmeans_cluster(ctx, cb.Cloud(ctx, pts), cent0, max_iter=max_iter, tol=tol)
    rc, rl, rit = kf.lloyd(pts, cent0, max_iter, tol)
    assert res["iterations"] == rit
    assert np.array_equal(res["labels"], rl)
    assert _same_f32(res["centroids"], rc)
    if case == "max_iter_0":
        assert rit == 0 and not rl.any() and _same_f32(res["centroids"], cent0)


def test_assign_point_whose_distances_all_overflow_gets_label_0(cb, ctx):
    rng = np.random.default_rng(3)
    cent = kr.dyadic(rng, (40, 3), 3.0)
    pts = np.vstack([kr.dyadic(rng, (500, 3), 3.0), [[3e19, 0, 0], [0, -3e19, 3e19]]]).astype(np.float32)
    labels, sums, counts = cb.kmeans_assign(ctx, cb.Cloud(ctx, pts), cent)
    want = kf.assign(pts, cent)
    assert np.array_equal(labels, want) and labels[-2:].tolist() == [0, 0]
    ws, wc = kf.sums(pts, want, 40)
    assert np.array_equal(counts, wc) and np.array_equal(sums[1:], ws[1:])  # cluster 0's double sum rounds


def _with_bad_rows(pts, rng):
    """pts with kr.BAD_ROWS (twice) inserted at random positions; returns (pts, mask of the finite rows)."""
    n, k = len(pts), 2 * len(kr.BAD_ROWS)
    pos = rng.choice(n + k, size=k, replace=False)
    keep = np.ones(n + k, bool)
    keep[pos] = False
    full = np.empty((n + k, 3), np.float32)
    full[keep] = pts
    full[np.sort(pos)] = np.concatenate([kr.BAD_ROWS, kr.BAD_ROWS])
    return full, keep


@pytest.mark.parametrize("case", ["uniform", "cluster0_largest_and_repaired", "global_sums"])
def test_nonfinite_points_are_inert(cb, ctx, case):
    """NaN / Inf rows keep label 0, add nothing to any sum or count and are never the farthest member: the run
    equals the run on the cloud without them."""
    rng = np.random.default_rng(11)
    pts = kr.dyadic(rng, (8000 if case == "global_sums" else 3000, 3), 1.0)
    if case == "uniform":
        cent0, max_iter = kr.dyadic(rng, (16, 3), 1.0), 5
    elif case == "cluster0_largest_and_repaired":
        # cluster 0 holds most points and cluster 2 is empty: the repair searches cluster 0
        cent0, max_iter = np.array([[0, 0, 0], [0.875, 0.875, 0.875], [50, 50, 50]], np.float32), 3
    else:  # K = 5889: global sums, hundreds of repairs
        cent0, max_iter = kr.dyadic(rng, (5889, 3), 1.0), 2
    dirty, keep = _with_bad_rows(pts, rng)
    labels, sums, counts = cb.kmeans_assign(ctx, cb.Cloud(ctx, dirty), cent0)
    ws, wc = kf.sums(pts, kf.assign(pts, cent0), len(cent0))
    assert np.array_equal(counts, wc) and np.array_equal(sums, ws)
    assert not labels[~keep].any()

    got = cb.kmeans_cluster(ctx, cb.Cloud(ctx, dirty), cent0, max_iter=max_iter, tol=0.0)
    clean = cb.kmeans_cluster(ctx, cb.Cloud(ctx, pts), cent0, max_iter=max_iter, tol=0.0)
    rc, rl, rit = kf.lloyd(pts, cent0, max_iter, 0.0)
    assert got["iterations"] == clean["iterations"] == rit
    assert np.array_equal(got["labels"][keep], clean["labels"]) and np.array_equal(clean["labels"], rl)
    assert not got["labels"][~keep].any()
    assert _same_f32(got["centroids"], clean["centroids"]) and _same_f32(clean["centroids"], rc)
    assert np.isfinite(got["centroids"]).all()


def test_empty_cloud(cb, ctx):
    """n = 0: no device fault. The assignment finds nothing; the loop runs one iteration in which every cluster
    is empty and nothing can be repaired, so every centroid is 0 * (1 / 0) = NaN, then stops (no label changed).
    Empty vector sets behave the same in every D, also from a null pointer (the data of an empty container)."""
    cent0 = np.array([[0, 0, 0], [1, 1, 1], [2, 2, 2]], np.float32)
    for empty in (cb.Cloud(ctx, np.zeros((0, 3), np.float32)), cb.Vectors(ctx, device_ptr=0, n=0, D=3),
                  cb.Vectors(ctx, device_ptr=0, n=0, D=2)):
        c0 = np.ascontiguousarray(cent0[:, :getattr(empty, "D", 3)])
        labels, sums, counts = cb.kmeans_assign(ctx, empty, c0)
        assert labels.shape == (0,) and not sums.any() and not counts.any()
        for tol in (0.0, 1e-3):
            res = cb.kmeans_cluster(ctx, empty, c0, max_iter=10, tol=tol)
            assert res["iterations"] == 1 and np.isnan(res["centroids"]).all() and res["labels"].shape == (0,)
            rc, _, rit = kf.lloyd(np.zeros((0, c0.shape[1]), np.float32), c0, 10, tol)
            assert rit == 1 and np.isnan(rc).all()
