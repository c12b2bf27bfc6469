"""GPU parity: cb_cloud_estimate_normals_mcd (NormalEstimation with MinimumCovarianceDeterminant) against the serial
restatement of oracle/robust_normals_oracle.cpp on brute-force neighbourhoods (ascending (d2, index), the kernel's
order).

Bars: status and covariance (cov6) bit-identical, NaN pattern identical. The normal and the curvature come from the
plain path's eigen step, which is not pinned against the oracle's double Jacobi (DESIGN §6): normals within
1 - |n.n_ref| < 1e-5 where the eigenvalue gap is clear, on the oracle's side of the view point or the reference normals,
curvature within 1e-4. Against cb_cloud_estimate_normals (the same eigen step on the device), h == size is bit for bit.
"""
import ctypes as C
import gc

import numpy as np
import pytest

from cilantro_b200 import capi, synth
from oracle import robust_normals as orn

pytestmark = pytest.mark.gpu

CB_ERR_INVALID, CB_ERR_UNSUPPORTED = -1, -5  # include/cilantro_b200.h
RECIPE = dict(num_trials=2, num_refinements=1, chi_square_threshold=6.25)  # examples/robust_normal_estimation.cpp


def _scene(n, seed, outliers=0.1):
    """A noisy sheet with a share of points pushed off it (the outliers the chi-square test should catch)."""
    pts, nrm = synth.surface_cloud(n, seed=seed, noise=0.0005)
    rng = np.random.default_rng(seed + 100)
    off = rng.random(n) < outliers
    pts = pts.copy()
    pts[off] += (nrm[off] * rng.uniform(0.01, 0.03, (off.sum(), 1))).astype(np.float32)
    return pts, nrm, off


def _full(c6):
    return np.stack([c6[:, [0, 1, 2]], c6[:, [1, 3, 4]], c6[:, [2, 4, 5]]], axis=1).astype(np.float64)


def _compare(got, want, pts, view_point=None, ref_normals=None):
    assert np.array_equal(got["status"], want["status"]), np.flatnonzero(got["status"] != want["status"])[:10]
    ok = want["status"] == 0
    assert np.array_equal(np.isnan(got["normals"]).any(axis=1), ~ok)
    assert np.array_equal(np.isnan(got["curvature"]), np.isnan(want["curvature"]))  # (a zero covariance: 0 / 0)
    assert np.array_equal(got["cov6"].view(np.uint32), want["cov6"].view(np.uint32)), "covariance not bit-identical"
    if not ok.any():
        return
    w = np.linalg.eigvalsh(_full(want["cov6"][ok]))
    well = (w[:, 1] - w[:, 0]) / np.maximum(np.abs(w[:, 2]), 1e-30) > 1e-2
    g, r = got["normals"][ok][well].astype(np.float64), want["normals"][ok][well].astype(np.float64)
    dots = np.sum(g * r, axis=1)
    assert np.all(1 - np.abs(dots) < 1e-5), np.max(1 - np.abs(dots))
    if ref_normals is not None or view_point is not None:
        e = (ref_normals[ok][well].astype(np.float64) if ref_normals is not None else
             np.asarray(view_point, np.float64) - pts[ok][well].astype(np.float64))
        side = np.sum(r * e, axis=1)
        decided = np.abs(side) > 1e-4 * np.linalg.norm(e, axis=1)
        assert np.all(dots[decided] > 0)
    assert np.allclose(got["curvature"][ok][well], want["curvature"][ok][well], atol=1e-4, equal_nan=True)


@pytest.mark.parametrize("k", [3, 4, 8, 12, 16, 32, 33, 64, 128])
def test_mcd_bit_identical_to_oracle(ctx, k):
    pts, _, _ = _scene(3000 if k <= 33 else 1500, seed=k)
    cloud = capi.Cloud(ctx, pts)
    nb = orn.estimate_normals_mcd(pts, k=k, num_trials=1, num_refinements=0)
    neighbors = (nb["nbr"], nb["cnt"])
    vp = [0.5, 0.5, 5.0]
    for trials, refinements in ((1, 0), (2, 1), (6, 3)):
        for ratio in (0.5, 0.75, 1.0):
            for chi2 in (-1.0, 6.25):
                kw = dict(num_trials=trials, num_refinements=refinements, inlier_ratio=ratio, chi_square_threshold=chi2,
                          seed=k)
                got = cloud.estimate_normals_mcd(k=k, view_point=vp, want_cov=True, **kw)
                want = orn.estimate_normals_mcd(pts, k=k, view_point=vp, neighbors=neighbors, **kw)
                _compare(got, want, pts, view_point=vp)


def test_mcd_knn_in_radius_and_reference_normals(ctx):
    pts, nrm, _ = _scene(8000, seed=3)
    r2 = float(np.float32(0.02**2))
    got = capi.Cloud(ctx, pts).estimate_normals_mcd(k=16, radius2=r2, want_cov=True, seed=4, **RECIPE)
    want = orn.estimate_normals_mcd(pts, k=16, radius2=r2, seed=4, **RECIPE)
    assert (want["cnt"] < 3).any() and (want["cnt"] == 16).any() and ((want["cnt"] > 3) & (want["cnt"] < 16)).any()
    assert set(np.unique(want["status"])) >= {0, 1, 2}
    _compare(got, want, pts)
    rng = np.random.default_rng(5)
    ref_n = rng.standard_normal(nrm.shape).astype(np.float32)
    got = capi.Cloud(ctx, pts, ref_n).estimate_normals_mcd(k=12, view_point=[0.5, 0.5, 5.0], use_current_as_ref=True,
                                                          want_cov=True, seed=4)
    want = orn.estimate_normals_mcd(pts, k=12, ref_normals=ref_n, seed=4)
    _compare(got, want, pts, ref_normals=ref_n)
    assert (np.sum(got["normals"] * ref_n, axis=1)[got["status"] == 0] >= 0).mean() > 0.999


def test_mcd_whole_neighbourhood_equals_plain_normals(ctx):
    pts, _, _ = _scene(20000, seed=8)
    vp = [0.5, 0.5, 5.0]
    for k, ratio in ((3, 0.75), (12, 1.0), (40, 0.99), (128, 1.0)):
        cloud = capi.Cloud(ctx, pts)
        plain = cloud.estimate_normals(k=k, view_point=vp, want_cov=True)
        got = cloud.estimate_normals_mcd(k=k, view_point=vp, inlier_ratio=ratio, want_cov=True)
        assert (got["status"] == 0).all()
        for key in ("normals", "curvature", "cov6"):
            assert np.array_equal(got[key].view(np.uint32), plain[key].view(np.uint32)), (k, key)
    # the normals stay on the device: downloading the cloud gives them back
    _, dn = cloud.download(normals=True)
    assert np.array_equal(dn.view(np.uint32), got["normals"].view(np.uint32))


def test_mcd_seed_reproducible_across_calls_and_contexts(ctx):
    pts, _, _ = _scene(10000, seed=12)
    a = capi.Cloud(ctx, pts).estimate_normals_mcd(k=12, want_cov=True, seed=99)
    b = capi.Cloud(ctx, pts).estimate_normals_mcd(k=12, want_cov=True, seed=99)
    ctx2 = capi.Context(0)
    try:
        c = capi.Cloud(ctx2, pts).estimate_normals_mcd(k=12, want_cov=True, seed=99)
    finally:
        ctx2.close()
    for other in (b, c):
        assert np.array_equal(a["cov6"].view(np.uint32), other["cov6"].view(np.uint32))
        assert np.array_equal(a["normals"].view(np.uint32), other["normals"].view(np.uint32))
    d = capi.Cloud(ctx, pts).estimate_normals_mcd(k=12, want_cov=True, seed=100)
    changed = np.any(a["cov6"].view(np.uint32) != d["cov6"].view(np.uint32), axis=1)
    assert changed.mean() > 0.5, changed.mean()


def test_mcd_edges(ctx):
    kw = dict(want_cov=True, **RECIPE)
    empty = capi.Cloud(ctx, np.zeros((0, 3), np.float32)).estimate_normals_mcd(k=8, **kw)
    assert empty["status"].size == 0
    two = capi.Cloud(ctx, np.array([[0, 0, 0], [1, 0, 0]], np.float32)).estimate_normals_mcd(k=8, **kw)
    assert (two["status"] == 1).all() and np.isnan(two["normals"]).all()
    rng = np.random.default_rng(2)
    pts = rng.random((3000, 3), dtype=np.float32)
    pts[105:145] = pts[105]  # a fully coincident neighbourhood
    pts[::50] = np.nan
    pts[1::50] = np.inf
    pts[2::50] = pts[3::50]  # exact duplicates
    got = capi.Cloud(ctx, pts).estimate_normals_mcd(k=12, **kw)
    want = orn.estimate_normals_mcd(pts, k=12, **RECIPE)
    _compare(got, want, pts)
    assert (got["status"][::50] == 1).all() and (got["status"][1::50] == 1).all()
    # coincident: a (numerically) zero covariance has a finite determinant, so a trial qualifies; its inverse is not
    # finite, so the chi-square test rejects the point
    assert (got["status"][105:145] == 2).all()
    free = capi.Cloud(ctx, pts).estimate_normals_mcd(k=12, num_trials=2, num_refinements=1, want_cov=True)
    assert (free["status"][105:145] == 0).all() and (np.abs(free["cov6"][105:145]) < 1e-12).all()
    # covariances that overflow fp32: no trial has a finite determinant
    huge = (rng.random((2000, 3)) * 3e12).astype(np.float32)
    got = capi.Cloud(ctx, huge).estimate_normals_mcd(k=12, want_cov=True, num_trials=2, num_refinements=1)
    want = orn.estimate_normals_mcd(huge, k=12, num_trials=2, num_refinements=1)
    _compare(got, want, huge)
    assert (got["status"] == 3).mean() > 0.9


def test_mcd_rejected_arguments(ctx):
    cloud = capi.Cloud(ctx, np.random.default_rng(0).random((100, 3), dtype=np.float32))
    cases = [(dict(num_trials=0), CB_ERR_INVALID), (dict(num_refinements=-1), CB_ERR_INVALID),
             (dict(inlier_ratio=float("nan")), CB_ERR_INVALID), (dict(inlier_ratio=float("inf")), CB_ERR_INVALID),
             (dict(min_sample_size=1), CB_ERR_UNSUPPORTED), (dict(min_sample_size=33), CB_ERR_UNSUPPORTED),
             (dict(k=129), CB_ERR_UNSUPPORTED), (dict(k=0, radius2=0.01), CB_ERR_UNSUPPORTED),
             (dict(k=-1), CB_ERR_INVALID)]
    for kw, code in cases:
        args = dict(k=8)
        args.update(kw)
        with pytest.raises(capi.CbError) as e:
            cloud.estimate_normals_mcd(**args)
        assert f"error {code}:" in str(e.value), (kw, str(e.value))
    rc = capi.lib().cb_cloud_estimate_normals_mcd(ctx.h, cloud.h, C.c_int(8), C.c_float(0.0), None, C.c_int(0), None,
                                                  None, None, None, None, None)
    assert rc == CB_ERR_INVALID
    # min_sample_size at its bounds runs
    pts = cloud.download()
    for m in (2, 32):
        got = cloud.estimate_normals_mcd(k=64, min_sample_size=m, num_trials=1, num_refinements=1, want_cov=True)
        want = orn.estimate_normals_mcd(pts, k=64, min_sample_size=m, num_trials=1, num_refinements=1)
        _compare(got, want, pts)


def test_mcd_device_memory_returns_to_baseline(ctx):
    cu = C.CDLL("libcuda.so.1")
    dev, pool = C.c_int(), C.c_void_p()
    assert cu.cuDeviceGet(C.byref(dev), 0) == 0 and cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0

    def used():
        ctx.synchronize()
        v = C.c_uint64()
        assert cu.cuMemPoolGetAttribute(pool, 7, C.byref(v)) == 0  # CU_MEMPOOL_ATTR_USED_MEM_CURRENT
        return v.value

    pts, _, _ = _scene(20000, seed=30)
    cloud = capi.Cloud(ctx, pts)
    cloud.estimate_normals_mcd(k=12, want_cov=True)  # allocates the cloud's normal buffers once
    gc.collect()  # objects of earlier tests on the shared context
    base = used()
    for i in range(100):
        cloud.estimate_normals_mcd(k=12 + i % 3, want_cov=i % 2 == 0, seed=i)
        if i % 10 == 0:
            with pytest.raises(capi.CbError):
                cloud.estimate_normals_mcd(k=8, num_trials=0)
    gc.collect()
    assert used() == base


def test_robust_normals_feed_combined_icp(ctx, orc):
    """downsample -> robust normals -> drop the invalid ones -> SimpleCombinedMetricRigidICP3f, on the device."""
    dst, _ = synth.surface_cloud(40000, seed=6, noise=0.0005)
    T_ref = synth.rigid_from_axis_angle([1, 2, -1], 0.01, [0.004, -0.003, 0.002])
    src = synth.apply(synth.invert(T_ref), dst[:20000]).astype(np.float32)
    d = capi.Cloud(ctx, dst).grid_downsample(0.005)
    rob = d.estimate_normals_mcd(k=12, view_point=[0.5, 0.5, 10.0], **RECIPE)
    keep = rob["status"] == 0
    assert 0.5 < keep.mean() < 1.0
    pts = d.download()[keep]  # PointCloud3f::removeInvalidNormals()
    nrm = rob["normals"][keep]
    kw = dict(metric="combined", max_iter=12, tol=0.0, max_d2=np.float32(0.02**2), w_pt=0.1, w_pl=1.0)
    res = capi.Icp(ctx, capi.Cloud(ctx, pts, nrm), capi.Cloud(ctx, src)).estimate(**kw)
    ref = orc.icp(pts, src, orc.make_knn(pts), dst_n=nrm, **kw)
    assert res["iterations"] == ref["iterations"]
    assert synth.frobenius(res["T"], ref["T"]) < 1e-5
    assert synth.frobenius(res["T"], T_ref) < 2e-3
