"""Feature-space correspondence search of the rigid ICP on the device (cb_icp_set_features) against the CPU restatement
(oracle/feature_icp_oracle.cpp: brute-force search on nanoflann's L2 arithmetic, the main oracle's filters, estimators
and loop): correspondence lists identical (indices, value bits, order) for every feature kind and engine option, with a
finite radius and unbounded, on clouds with outliers far outside the grid (the far-sweep path); transforms within 1e-5
over 12 iterations; the identities with the point-only path; the value of colour on a textured sheet; the edges."""
import ctypes as C
import gc

import numpy as np
import pytest

from cilantro_b200 import capi, synth
from conftest import frob

pytestmark = pytest.mark.gpu

FLT_MAX = float(np.finfo(np.float32).max)
KINDS = ["point_normal", "point_color", "point_normal_color"]
MODES = {
    "s2f": {},
    "f2s": dict(search_dir="first_to_second"),
    "both": dict(search_dir="both"),
    "both_reciprocal": dict(search_dir="both", require_reciprocal=True),
    "fraction": dict(inlier_fraction=0.8),
    "one_to_one": dict(one_to_one=True),
}
W_N, W_C = 0.5, 5.0  # the reference example's PointNormalColorFeaturesAdaptor3f weights


@pytest.fixture(scope="module")
def F(orc):
    from oracle import feature_icp

    feature_icp.build()
    return feature_icp


def _scene(n, seed, outliers=True):
    s = synth.textured_sheet_pair(n, seed=seed)
    if outliers:  # far outside both grids: their searches run the far sweep (unbounded) or find nothing
        far = np.array([[40.0, 40.0, 40.0], [-25.0, 3.0, 0.5], [0.5, 0.5, 60.0]], np.float32)
        for key in ("dst", "src"):
            s[key] = np.vstack([s[key], far + (0.5 if key == "src" else 0.0)]).astype(np.float32)
        for key in ("dst_normals", "src_normals"):
            s[key] = np.vstack([s[key], np.tile([[0.0, 0.0, 1.0]], (3, 1))]).astype(np.float32)
        for key in ("dst_colors", "src_colors"):
            s[key] = np.vstack([s[key], np.full((3, 3), 0.5)]).astype(np.float32)
    return s


def _arrays(kind, s):
    nrm = "normal" in kind
    col = "color" in kind
    return dict(dst_normals=s["dst_normals"] if nrm else None, dst_colors=s["dst_colors"] if col else None,
                src_normals=s["src_normals"] if nrm else None, src_colors=s["src_colors"] if col else None)


def _tails(F, kind, s, w_n=W_N, w_c=W_C):
    a = _arrays(kind, s)
    return (F.tails(kind, a["dst_normals"], a["dst_colors"], w_n, w_c),
            F.tails(kind, a["src_normals"], a["src_colors"], w_n, w_c))


def _icp(ctx, kind, s, w_n=W_N, w_c=W_C, src_normals_on_cloud=False):
    icp = capi.Icp(ctx, capi.Cloud(ctx, s["dst"], s["dst_normals"]),
                   capi.Cloud(ctx, s["src"], s["src_normals"] if src_normals_on_cloud else None))
    if kind != "point":
        icp.set_features(kind, normal_weight=w_n, color_weight=w_c, **_arrays(kind, s))
    return icp


T0 = np.array([[0.9998, -0.0175, 0.0, 0.025], [0.0175, 0.9998, 0.0, -0.015], [0.0, 0.0, 1.0, 0.0005]], np.float32)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("max_d2", [0.02, FLT_MAX])
def test_lists_match_oracle(ctx, F, kind, mode, max_d2):
    s = _scene(3000, seed=11)
    icp = _icp(ctx, kind, s)
    icp.estimate(metric="p2p", max_iter=1, tol=0.0, max_d2=max_d2, T_init=T0, **MODES[mode])
    f, sec, v = icp.correspondences()
    dt, st = _tails(F, kind, s)
    of, os_, ov = F.engine_correspondences(kind, s["dst"], dt, s["src"], st, T0, max_d2, **MODES[mode])
    assert len(f) > 0
    assert np.array_equal(f, of) and np.array_equal(sec, os_), (kind, mode, len(f), len(of))
    assert np.array_equal(v.view(np.uint32), ov.view(np.uint32))
    # the value is the feature distance: at least the xyz part of the pair
    q = synth.apply(T0, s["src"][sec]).astype(np.float64)
    assert np.all(v.astype(np.float64) >= ((q - s["dst"][f]) ** 2).sum(1) * (1 - 1e-5))


@pytest.mark.parametrize("kind", ["point_color", "point_normal_color"])
@pytest.mark.parametrize("cfg", [dict(metric="p2p"),
                                 dict(metric="combined", w_pt=0.1, w_pl=1.0),
                                 dict(metric="combined", w_pt=0.1, w_pl=1.0, pt_rbf_sigma=0.5, pl_rbf_sigma=0.3),
                                 dict(metric="p2p", search_dir="both", require_reciprocal=True, inlier_fraction=0.9)])
def test_loop_matches_oracle(ctx, F, kind, cfg):
    s = _scene(4000, seed=5)
    kw = dict(max_iter=12, tol=0.0, max_d2=0.05)
    got = _icp(ctx, kind, s).estimate(**kw, **cfg)
    dt, st = _tails(F, kind, s)
    want = F.icp(kind, s["dst"], dt, s["src"], st, dst_n=s["dst_normals"], **kw, **cfg)
    assert got["iterations"] == want["iterations"] == 12
    assert got["num_corr"] == want["num_corr"]
    assert frob(got["T"], want["T"]) < 1e-5, frob(got["T"], want["T"])
    # with the default tolerance the two stop after the same number of iterations
    kw["tol"] = 1e-5
    got = _icp(ctx, kind, s).estimate(**kw, **cfg)
    want = F.icp(kind, s["dst"], dt, s["src"], st, dst_n=s["dst_normals"], **kw, **cfg)
    assert (got["iterations"], got["num_corr"]) == (want["iterations"], want["num_corr"])
    assert frob(got["T"], want["T"]) < 1e-5


@pytest.mark.parametrize("mode", ["s2f", "f2s", "both", "one_to_one"])
def test_zero_color_weight_is_the_point_search(ctx, mode):
    """[p, 0 c]: every tail term is +0, so the feature distance is the xyz distance bit for bit."""
    s = _scene(3000, seed=3)
    kw = dict(metric="p2p", max_iter=1, tol=0.0, max_d2=0.02, T_init=T0, **MODES[mode])
    a, b = _icp(ctx, "point_color", s, w_c=0.0), _icp(ctx, "point", s)
    a.estimate(**kw)
    b.estimate(**kw)
    for x, y in zip(a.correspondences(), b.correspondences()):
        assert np.array_equal(np.asarray(x).view(np.uint32 if x.dtype == np.float32 else np.int64),
                              np.asarray(y).view(np.uint32 if y.dtype == np.float32 else np.int64))
    kw["max_iter"] = 8
    ra, rb = a.estimate(**kw), b.estimate(**kw, host_loop=True)
    if mode != "s2f":  # both on the list path: the same kernels over the same list
        assert np.array_equal(ra["T"].view(np.uint32), rb["T"].view(np.uint32))
    else:  # the point-only default runs the fused search + accumulation: same pairs, another summation order
        assert frob(ra["T"], rb["T"]) < 1e-6
    assert (ra["iterations"], ra["num_corr"]) == (rb["iterations"], rb["num_corr"])


def test_point_kind_restores_the_default_path(ctx):
    s = _scene(5000, seed=8, outliers=False)
    # started at the registering transform, the point-only run converges and stays on the device loop
    kw = dict(metric="combined", w_pt=0.1, w_pl=1.0, max_iter=10, tol=0.0, max_d2=0.02, T_init=s["T_ref"])
    icp = _icp(ctx, "point_normal_color", s)
    icp.estimate(**kw)
    icp.set_features("point")
    got = icp.estimate(**kw)
    fresh = _icp(ctx, "point", s).estimate(**kw)
    assert np.array_equal(got["T"].view(np.uint32), fresh["T"].view(np.uint32))
    assert (got["iterations"], got["num_corr"]) == (fresh["iterations"], fresh["num_corr"])
    icp.loop_cache()  # raises unless the run was on the device-resident loop


def test_color_recovers_the_in_plane_offset(ctx):
    """A low-relief textured sheet shifted in-plane by (0.03, -0.02): the geometry barely constrains the shift, the colours
    do. On the CPU restatement (20 000 points, seed 4) the coloured ICP ends within ~1e-3 of the shift and the point-only
    ICP ~2.5e-2 away from it."""
    s = synth.textured_sheet_pair(20000, seed=4)
    kw = dict(metric="combined", w_pt=0.1, w_pl=1.0, max_iter=30, tol=1e-6, max_d2=0.02)
    col = _icp(ctx, "point_color", s, w_c=0.5).estimate(**kw)
    pt = _icp(ctx, "point", s).estimate(**kw)
    err_col = float(np.linalg.norm(col["T"][:2, 3] - s["T_ref"][:2, 3]))
    err_pt = float(np.linalg.norm(pt["T"][:2, 3] - s["T_ref"][:2, 3]))
    print(f"in-plane offset error: coloured {err_col:.2e}, point-only {err_pt:.2e}")
    assert err_col < 2e-3 and err_pt > 1.5e-2, (err_col, err_pt)


def test_non_finite_tails_are_inert(ctx, F):
    s = _scene(3000, seed=2)
    rng = np.random.default_rng(0)
    bad_src, bad_dst = rng.choice(3000, 50, replace=False), rng.choice(3000, 50, replace=False)
    s["src_colors"][bad_src[:25], 1] = np.nan
    s["src_normals"][bad_src[25:], 0] = np.inf
    s["dst_colors"][bad_dst[:25], 2] = np.nan
    s["dst_normals"][bad_dst[25:], 2] = -np.inf
    for mode in ("s2f", "both"):
        icp = _icp(ctx, "point_normal_color", s)
        icp.estimate(metric="p2p", max_iter=1, tol=0.0, max_d2=FLT_MAX, T_init=T0, **MODES[mode])
        f, sec, v = icp.correspondences()
        assert not np.isin(sec, bad_src).any() and not np.isin(f, bad_dst).any() and np.isfinite(v).all()
        dt, st = _tails(F, "point_normal_color", s)
        of, os_, ov = F.engine_correspondences("point_normal_color", s["dst"], dt, s["src"], st, T0, FLT_MAX,
                                               **MODES[mode])
        assert np.array_equal(f, of) and np.array_equal(sec, os_) and np.array_equal(v.view(np.uint32), ov.view(np.uint32))


def test_empty_clouds_behave_as_the_point_path(ctx):
    e = np.zeros((0, 3), np.float32)
    s = _scene(500, seed=1, outliers=False)
    for dst, src in ((e, s["src"]), (s["dst"], e)):
        icp = capi.Icp(ctx, capi.Cloud(ctx, dst), capi.Cloud(ctx, src))
        icp.set_features("point_color", dst_colors=np.zeros_like(dst), src_colors=np.zeros_like(src))
        res = icp.estimate(metric="p2p", max_iter=3, tol=0.0, max_d2=0.02)
        ref = capi.Icp(ctx, capi.Cloud(ctx, dst), capi.Cloud(ctx, src)).estimate(metric="p2p", max_iter=3, tol=0.0,
                                                                                max_d2=0.02, host_loop=True)
        assert res["num_corr"] == 0 and np.array_equal(res["T"], ref["T"]) and res["iterations"] == ref["iterations"]
        assert len(icp.correspondences()[0]) == 0


def test_rejected_arguments(ctx):
    s = _scene(500, seed=1, outliers=False)
    icp = _icp(ctx, "point", s)
    lib = capi.lib()
    c = capi._p(s["dst_colors"])
    n = capi._p(s["dst_normals"])
    for args in ((2, None, None, None, c, 1.0, 1.0),     # no dst colours
                 (1, n, None, None, None, 1.0, 1.0),     # no src normals
                 (3, n, c, n, None, 1.0, 1.0),           # no src colours
                 (2, None, c, None, c, 1.0, float("nan")),
                 (1, n, None, n, None, float("inf"), 1.0),
                 (3, n, c, n, c, 1.0, float("-inf")),
                 (4, n, c, n, c, 1.0, 1.0)):             # no such kind
        rc = lib.cb_icp_set_features(icp.h, C.c_int(args[0]), args[1], args[2], args[3], args[4], C.c_float(args[5]),
                                     C.c_float(args[6]))
        assert rc == -1, args  # CB_ERR_INVALID
    # an unused weight may be anything; an unused array may be NULL
    assert lib.cb_icp_set_features(icp.h, C.c_int(2), None, c, None, c, C.c_float(float("nan")), C.c_float(1.0)) == 0


def test_create_set_estimate_destroy_cycles_return_device_memory(ctx):
    import torch

    s = _scene(3000, seed=6)
    dst = capi.Cloud(ctx, s["dst"], s["dst_normals"])
    src = capi.Cloud(ctx, s["src"])

    def cycle():
        icp = capi.Icp(ctx, dst, src)
        icp.set_features("point_normal_color", normal_weight=W_N, color_weight=W_C, **_arrays("point_normal_color", s))
        icp.estimate(metric="p2p", max_iter=2, tol=0.0, max_d2=0.02, search_dir="both")
        icp.close()

    cycle()
    ctx.synchronize()
    gc.collect()
    free0 = torch.cuda.mem_get_info(0)[0]
    for _ in range(100):
        cycle()
    ctx.synchronize()
    gc.collect()
    free1 = torch.cuda.mem_get_info(0)[0]
    assert free1 >= free0 - (2 << 20), (free0, free1)


@pytest.mark.parametrize("kind", ["point_color", "point_normal_color"])
def test_accumulate_sums_over_the_feature_list(ctx, F, kind):
    """cb_icp_accumulate with features: the Kabsch moments of the feature search's list (as the oracle lists it); after
    set_features("point") it accumulates over the xyz search again and the correspondences follow."""
    import oracle

    s = _scene(3000, seed=9)
    icp = _icp(ctx, kind, s)
    sums = icp.accumulate(T0, metric="p2p", max_d2=0.05)
    dt, st = _tails(F, kind, s)
    f, sec, v = F.engine_correspondences(kind, s["dst"], dt, s["src"], st, T0, 0.05)
    d = s["dst"][f].astype(np.float64)
    q = oracle.transform_points(T0, s["src"])[sec].astype(np.float64)
    want = np.concatenate([[len(f)], d.sum(0), q.sum(0), (d.T @ q).reshape(-1)])
    assert sums[0] == len(f)
    assert np.allclose(sums, want, rtol=1e-9, atol=1e-9)
    gf, gs, gv = icp.correspondences()
    assert np.array_equal(gf, f) and np.array_equal(gs, sec) and np.array_equal(gv.view(np.uint32), v.view(np.uint32))
    # back to the xyz search: the moments and the list are the point-only ones
    icp.set_features("point")
    sums_pt = icp.accumulate(T0, metric="p2p", max_d2=0.05)
    fresh = _icp(ctx, "point", s)
    assert np.array_equal(sums_pt, fresh.accumulate(T0, metric="p2p", max_d2=0.05))
    for x, y in zip(icp.correspondences(), fresh.correspondences()):
        assert np.array_equal(x, y)
