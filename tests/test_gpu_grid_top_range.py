"""Grid searches at the top of the fp32 range against brute force (orc.BruteKnn, the fp32 arithmetic contract): clouds
whose neighbour structure lies along z while x and y sit in [2^126, FLT_MAX], a cloud whose extent forces the grid
origin up from one cell below the box, and a cloud spanning nearly +-FLT_MAX, which no fp32 cell coordinate can hold
and whose index build is refused. Indices and counts identical, d2 and covariances bit-identical; ICP's warp-pooled
pass (accumulate) and per-lane pass (residuals) must agree with brute force and so with each other."""
import time

import numpy as np
import pytest

from test_gpu_grid_edges import _bits, _check
from top_range_ref import FMAX, GUARD, raised_origin_cloud, top_range_cloud, top_range_queries, wide_cloud

pytestmark = pytest.mark.gpu

F32 = np.float32
KS = (1, 16, 256)


def _nan_bits(a):
    """Bit patterns with every NaN as one value (the NaN a GPU creates differs from x86's)."""
    a = np.ascontiguousarray(a, F32)
    return np.where(np.isnan(a), np.uint32(0x7fc00000), a.view(np.uint32))


@pytest.mark.parametrize("which", ["top", "raised_origin"])
def test_searches_at_the_top_of_the_range(cb, ctx, orc, which):
    t0 = time.perf_counter()
    pts = top_range_cloud() if which == "top" else raised_origin_cloud()
    qry = top_range_queries(pts)
    cl = cb.Cloud(ctx, pts)
    info = cl.grid_info()
    d2 = orc.BruteKnn(pts).neighborhoods(pts, 2, FMAX)[1][:, 1]
    assert (d2 == 0).any() and (d2 == F32(0.25) ** 2).any()  # duplicates, and lattice neighbours
    if which == "top":
        assert (np.abs(qry.astype(np.float64)).sum(axis=1) >= GUARD).sum() > len(pts) // 2
    else:  # one cell below the box would put its far side beyond FLT_MAX of the origin
        x = pts[:, 0].astype(np.float64)
        assert x.max() - (x.min() - info["cell_edge"]) > FMAX
    out = _check(cb, ctx, orc, pts, qry, max_d2=FMAX, ks=KS, r2=F32(1.0), corr_d2=F32(0.25) ** 2, ref=cl)
    assert (out["knn1"][0] >= 0).sum() >= len(pts)  # every cloud point finds itself or a twin
    assert (out["radius"][2] < 1.0).all() and np.diff(out["radius"][0]).max() > 1
    # a pair exactly at the bound: d2 == 1 is in the lattice and must stay out
    assert (orc.BruteKnn(pts).neighborhoods(pts, 16, FMAX)[1] == 1.0).any()
    # the same queries on the bound itself
    _check(cb, ctx, orc, pts, qry, max_d2=F32(1.0), ks=(16,), ref=cl)
    print(f"[top-range] {which}: grid_info {info}, {time.perf_counter() - t0:.3f} s")


def test_normals_at_the_top_of_the_range(cb, ctx, orc):
    pts = top_range_cloud(nz=24, dups=10)
    for k in (4, 16):
        got = cb.Cloud(ctx, pts).estimate_normals(k=k, view_point=[0.5, 0.5, 10.0], want_cov=True)
        want = orc.estimate_normals(pts, orc.BruteKnn(pts), k=k, view_point=[0.5, 0.5, 10.0])
        assert np.array_equal(_nan_bits(got["cov6"]), _nan_bits(want[2])), f"k={k}: covariances differ"


def test_icp_passes_at_the_top_of_the_range(cb, ctx, orc):
    """accumulate runs the pooled search of the ICP pass, residuals the per-lane one, on the same queries."""
    dst = top_range_cloud(seed=4)
    src = top_range_queries(dst, seed=5)
    src = src[np.isfinite(src).all(axis=1)]
    I = np.eye(3, 4, dtype=F32)
    knn = orc.BruteKnn(dst)
    icp = cb.Icp(ctx, cb.Cloud(ctx, dst), cb.Cloud(ctx, src))
    for max_d2 in (F32(0.25) ** 2, F32(1.0), F32(FMAX)):
        sums = icp.accumulate(I, metric="p2p", max_d2=max_d2)
        i1, i2, v = orc.find_correspondences(I, src, knn, max_d2)
        assert int(sums[0]) == i1.size, (max_d2, sums[0], i1.size)
        assert i1.size > len(dst) // 2
    got = icp.residuals(I, metric="p2p")
    # queries with a neighbour at a finite d2 (the oracle's residual is defined only for those); the rest get NaN
    has = knn.query(src, FMAX)[0] >= 0
    assert 0 < (~has).sum() < 10
    want = orc.icp_residuals(dst, src[has], I, knn, metric="p2p")
    assert np.array_equal(_bits(got[has]), _bits(want)), f"{(_bits(got[has]) != _bits(want)).sum()} residuals differ"
    assert np.isnan(got[~has]).all() and (got == 0).sum() >= len(dst)


def test_cloud_spanning_nearly_all_of_fp32_is_refused(cb, ctx, orc):
    """x - origin of a cloud spanning more than FLT_MAX overflows for some of its points: the index build says so
    (CB_ERR_UNSUPPORTED) instead of searching inexactly, on every entry point that builds the index."""
    pts = wide_cloud()
    x = pts[:, 0].astype(np.float64)
    assert x.max() - x.min() > FMAX
    cl = cb.Cloud(ctx, pts)
    with pytest.raises(cb.CbError, match="-5"):
        cb.knn1_radius(ctx, cl, cl)
    with pytest.raises(cb.CbError, match="-5"):
        cb.Cloud(ctx, pts).segment(k=4)
    with pytest.raises(cb.CbError, match="-5"):
        cb.Cloud(ctx, pts).mean_shift(1.0, 3, 0.5)
    # the same cloud without its high cluster is searched
    half = pts[x < 0]
    _check(cb, ctx, orc, half, half, max_d2=FMAX, ks=(4,), ref=cb.Cloud(ctx, half))

