"""cb_cloud_mean_shift at its edges, bit for bit against the oracle (oracle/mean_shift.py) and, on the small inputs, the
numpy restatement (mean_shift_ref.py): the clustering alone (max_iter = 0) with pairs exactly at cluster_tol, a permuted
dense lattice that takes many rounds, signed zeros among bit-identical copies; cluster_tol, kernel_radius and
convergence_tol at their special values; seeds and points at the top of the fp32 range. Dyadic inputs throughout."""
import numpy as np
import pytest

import mean_shift_ref
from test_gpu_mean_shift import both, same
from top_range_ref import FMAX, top_range_cloud

pytestmark = pytest.mark.gpu

F32 = np.float32


@pytest.fixture(scope="module")
def ms():
    from oracle import mean_shift

    return mean_shift


def check(cb, ctx, ms, pts, *args, numpy_ref=False, **kw):
    got, want = both(cb, ctx, ms, pts, *args, **kw)
    same(got, want)
    if numpy_ref:
        r = mean_shift_ref.mean_shift(pts, *args, **kw)
        for k in ("offsets", "points", "point_to_cluster", "num_clusters", "iterations"):
            assert np.array_equal(got[k], r[k]), k
    return got


def test_clustering_alone_at_cluster_tol(cb, ctx, ms):
    """max_iter = 0: the seeds are clustered as given. Pairs 1 apart with cluster_tol 1 (d2 == tol^2, apart) and
    one ulp above 1 (together); chains 0.5 apart (every second seed a representative)."""
    rng = np.random.default_rng(1)
    base = np.column_stack([np.arange(300) * 8.0, np.zeros(300), np.zeros(300)])
    seeds = np.vstack([base, base + [0.0, 1.0, 0.0], base + [0.0, 0.0, 0.5], base + [0.0, 0.0, 1.0]])
    seeds = seeds[rng.permutation(len(seeds))].astype(F32)
    pts = seeds[:50]
    for tol in (1.0, float(np.nextafter(F32(1.0), F32(2.0))), 0.5, float(np.nextafter(F32(0.5), F32(1.0)))):
        got = check(cb, ctx, ms, pts, 1.0, 0, tol, seeds=seeds, numpy_ref=True)
        assert got["iterations"] == 0
        assert np.array_equal(got["shifted_seeds"].view(np.uint32), seeds.view(np.uint32))


def test_permuted_dense_lattice_takes_many_rounds(cb, ctx, ms):
    """A lattice at 0.625 cluster_tol in random seed order: whether a seed is a representative depends on chains of
    lower-index neighbours, so round_kernel runs many rounds."""
    g = np.arange(24, dtype=F32) * F32(0.625)
    seeds = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    seeds = seeds[np.random.default_rng(2).permutation(len(seeds))]
    got = check(cb, ctx, ms, seeds[:100], 1.0, 0, 1.0, seeds=seeds)
    assert 1 < got["num_clusters"] < len(seeds) // 2


def test_signed_zeros_and_bit_identical_copies(cb, ctx, ms):
    """+0.0 and -0.0 are different bit patterns (separate dedup groups) at distance 0, interleaved with exact copies."""
    z = np.array([[0.0, 0.0, 0.0], [-0.0, 0.0, 0.0], [0.0, -0.0, -0.0], [-0.0, -0.0, -0.0], [1.0, 0.0, -0.0]], F32)
    seeds = np.vstack([z[np.random.default_rng(3).integers(0, 5, 400)], z])
    assert len(np.unique(seeds.view(np.uint32), axis=0)) == 5
    for tol in (1.0, 1e-30, 0.0):
        check(cb, ctx, ms, seeds[:20], 0.5, 0, tol, seeds=seeds, numpy_ref=True)


@pytest.mark.parametrize("tol", [0.0, -1.0, 1e-30, 1.8e19, 2e19, np.inf, np.nan])
def test_cluster_tol_special_values(cb, ctx, ms, tol):
    """tol^2 underflowing to 0 (1e-30), near FLT_MAX (1.8e19), Inf (2e19, inf), negative and NaN; seeds up to 1e19 apart
    so that the large tolerances cluster some of them."""
    rng = np.random.default_rng(4)
    seeds = np.vstack([rng.integers(0, 4, (200, 3)) * 0.5, rng.integers(-2, 3, (40, 3)) * 2.0**62,
                       [[np.nan, 0, 0], [np.inf, 1, 1]]]).astype(F32)
    pts = rng.integers(0, 4, (100, 3)).astype(F32) * F32(0.5)
    if tol in (1.8e19, 2e19):
        with np.errstate(over="ignore"):
            t2 = F32(tol) * F32(tol)
        assert (t2 < np.inf) == (tol == 1.8e19)
    for max_iter in (0, 3):
        check(cb, ctx, ms, pts, 0.75, max_iter, tol, seeds=seeds)


def test_kernel_radius_and_convergence_tol_edges(cb, ctx, ms):
    rng = np.random.default_rng(5)
    pts = (rng.integers(0, 8, (300, 3)) * 0.25).astype(F32)
    seeds = pts[::3]
    # a radius exactly at lattice distances: 0.25 (d2 == r2, excluded), 0.5, and one ulp above each
    for r in (0.25, float(np.nextafter(F32(0.25), F32(1))), 0.5, float(np.nextafter(F32(0.5), F32(1)))):
        check(cb, ctx, ms, pts, r, 20, 0.1, seeds=seeds)
    check(cb, ctx, ms, pts[:40], np.inf, 5, 0.1, seeds=seeds, numpy_ref=True)  # every point in every window
    got = check(cb, ctx, ms, pts, -1.0, 5, 0.1, seeds=seeds)  # r^2 = 1 > 0: same as radius 1
    same(got, cb.Cloud(ctx, pts).mean_shift(1.0, 5, 0.1, seeds=seeds))
    for ctol in (0.0, np.nan, np.inf):
        got = check(cb, ctx, ms, pts, 0.5, 15, 0.1, convergence_tol=ctol, seeds=seeds)
        if ctol == np.inf:
            assert got["iterations"] == 1
        else:
            assert got["iterations"] > 1


def test_top_of_the_range(cb, ctx, ms):
    """Points and seeds with |x| + |y| + |z| >= 3e38: windows inside a column (x, y equal, d2 finite), bit-identical
    seeds there deduplicated, columns never merged (their d2 is Inf)."""
    pts = top_range_cloud(seed=6, nz=24, dups=20)
    seeds = np.vstack([pts[::2], pts[:30]])
    for r, it, tol in ((0.6, 10, 0.3), (1.0, 0, 0.3), (1.0, 0, 1e19), (2.0, 20, 2e19)):
        got = check(cb, ctx, ms, pts, r, it, tol, seeds=seeds, numpy_ref=it == 0)
        if it == 0 and tol == 0.3:
            assert got["num_clusters"] < len(seeds)  # bit-identical seeds share a cluster
    assert np.abs(pts).max() == FMAX
