"""ICP on inputs the uniform-cube pairs never produce: non-finite points, degenerate geometry (plane, line, coincident
points, a corridor) and cloud sizes at the block / reduction-group boundaries of the device passes.

Every case runs one iteration through the device-resident loop and through the host loop and compares the result with
tests/icp_ref.py (a float64 restatement of the step) on the product's own correspondences, which are first checked
against the oracle's; a few iterations are then compared between the loops and with the oracle. Where the rotation is
not unique (rank <= 1) the transform must be a proper rotation that maps the matched source points onto their
destinations. Each degenerate case asserts which branch of la::nearest_rotation (Newton polar iteration or Jacobi SVD)
its sigma takes.
"""
import numpy as np
import pytest

import icp_ref
from cilantro_b200 import synth
from conftest import frob

pytestmark = pytest.mark.gpu

ENGINE_KEYS = ("search_dir", "require_reciprocal", "one_to_one", "inlier_fraction")


def _is_engine(kw):
    return any(k in kw for k in ENGINE_KEYS)


def _pairs(cb, orc, icp, dst, src, T, max_d2, kw):
    """The product's correspondence list of the last search, checked against the oracle's on the same clouds."""
    f, s, _ = icp.correspondences()
    knn = orc.BruteKnn(dst)
    if _is_engine(kw):
        of, os_, _ = orc.engine_correspondences(dst, src, T, knn, max_d2, **{k: kw[k] for k in ENGINE_KEYS if k in kw})
    else:
        of, os_, _ = orc.find_correspondences(T, src, knn, max_d2)
    assert np.array_equal(f, of) and np.array_equal(s, os_)
    return f, s


def _ref_step(dst, src, T, f, s, metric, kw, dst_n=None, src_n=None):
    if metric == "p2p":
        return icp_ref.p2p_step(dst, src, T, f, s)
    fin_d, fin_s = icp_ref.finite_rows(dst), icp_ref.finite_rows(src)
    dm = dst[fin_d].astype(np.float64).mean(0).astype(np.float32)
    sm = src[fin_s].astype(np.float64).mean(0).astype(np.float32)
    return icp_ref.combined_step(dst, dst_n, src, T, f, s, kw.get("w_pt", 0.0), kw.get("w_pl", 1.0), dm, sm, src_n=src_n)


def _proper(T, tol=1e-5):
    R = np.asarray(T, np.float64)[:, :3]
    return abs(np.linalg.det(R) - 1) < tol and np.abs(R @ R.T - np.eye(3)).max() < tol


# ---- non-finite points ---------------------------------------------------------------------------------------------
BAD_ROWS = np.array([[np.nan, np.nan, np.nan], [np.inf, np.inf, np.inf], [-np.inf, -np.inf, -np.inf],
                     [np.inf, -np.inf, 0.5], [0.5, np.nan, 0.5], [-np.inf, 0.5, np.inf]], np.float32)


def _with_bad_rows(pts, nrm, rng):
    """pts with BAD_ROWS (twice) inserted at random positions; returns (pts, normals, index of each clean row)."""
    n = len(pts)
    k = 2 * len(BAD_ROWS)
    pos = np.sort(rng.choice(n + k, size=k, replace=False))
    keep = np.ones(n + k, bool)
    keep[pos] = False
    full = np.empty((n + k, 3), np.float32)
    full[keep] = pts
    full[pos] = np.concatenate([BAD_ROWS, BAD_ROWS])
    fn = None
    if nrm is not None:
        fn = np.empty((n + k, 3), np.float32)
        fn[keep] = nrm
        fn[pos] = [0.0, 0.0, 1.0]
    return full, fn, np.flatnonzero(keep)


NONFINITE_CONFIGS = [
    ("p2p", dict()),
    ("combined", dict(w_pt=0.1, w_pl=1.0)),
    ("symmetric", dict(w_pt=0.0, w_pl=1.0)),
    ("p2p", dict(search_dir="both")),
    ("p2p", dict(search_dir="both", require_reciprocal=True)),
    ("combined", dict(w_pt=0.1, w_pl=1.0, one_to_one=True)),
    ("p2p", dict(inlier_fraction=0.8)),
]


@pytest.mark.parametrize("where", ["dst", "src", "both"])
@pytest.mark.parametrize("cfg", range(len(NONFINITE_CONFIGS)),
                         ids=[m + "".join(f"-{k}" for k in kw if k not in ("w_pt", "w_pl")) for m, kw in NONFINITE_CONFIGS])
def test_nonfinite_points_are_inert(cb, ctx, orc, where, cfg):
    """NaN / Inf rows in either cloud change nothing: the result equals the run on the clouds without them (same
    correspondences, mapped back; same count; T within 1e-6). The pivot means skip them (DESIGN §6)."""
    metric, kw = NONFINITE_CONFIGS[cfg]
    dst, src, nrm, T_ref = synth.icp_pair(3000, seed=40 + cfg, noise=0.002, with_normals=True)
    src_n = (nrm.astype(np.float64) @ synth.invert(T_ref)[:, :3].T).astype(np.float32) if metric == "symmetric" else None
    rng = np.random.default_rng(cfg)
    dst_f, nrm_f, dmap = (_with_bad_rows(dst, nrm, rng) if where in ("dst", "both") else (dst, nrm, np.arange(len(dst))))
    src_f, srcn_f, smap = (_with_bad_rows(src, src_n, rng) if where in ("src", "both")
                           else (src, src_n, np.arange(len(src))))
    max_d2 = np.float32(0.03**2)
    pm = "p2p" if metric == "p2p" else "combined"
    clean = cb.Icp(ctx, cb.Cloud(ctx, dst, nrm), cb.Cloud(ctx, src, src_n))
    full = cb.Icp(ctx, cb.Cloud(ctx, dst_f, nrm_f), cb.Cloud(ctx, src_f, srcn_f))
    loops = (True,) if _is_engine(kw) else (False, True)
    for host_loop in loops:
        for iters in (1, 5):
            args = dict(metric=pm, max_iter=iters, tol=0.0, max_d2=max_d2, host_loop=host_loop, **kw)
            a = full.estimate(**args)
            b = clean.estimate(**args)
            assert np.isfinite(a["T"]).all(), (host_loop, iters, a["T"])
            assert a["num_corr"] == b["num_corr"] > 0, (host_loop, iters)
            assert frob(a["T"], b["T"]) < 1e-6, (host_loop, iters, frob(a["T"], b["T"]))
            fa, sa, _ = full.correspondences()
            fb, sb, _ = clean.correspondences()
            assert np.array_equal(fa, dmap[fb]) and np.array_equal(sa, smap[sb]), (host_loop, iters)
        # one iteration against the float64 step on the product's own pairs (checked against the oracle's)
        T0 = cb.identity()
        one = full.estimate(metric=pm, max_iter=1, tol=0.0, max_d2=max_d2, host_loop=host_loop, **kw)
        f, s = _pairs(cb, orc, full, dst_f, src_f, T0, max_d2, kw)
        Tr, _ = _ref_step(dst_f, src_f, T0, f, s, metric, kw, dst_n=nrm_f, src_n=srcn_f)
        assert frob(one["T"], Tr) < 2e-6, (host_loop, frob(one["T"], Tr))
    if metric == "p2p":  # the reference's point-to-point estimate uses the correspondences only: finite on these clouds
        want = orc.icp(dst_f, src_f, orc.BruteKnn(dst_f), metric="p2p", max_iter=5, tol=0.0, max_d2=max_d2, **kw)
        got = full.estimate(metric="p2p", max_iter=5, tol=0.0, max_d2=max_d2, **kw)
        assert got["num_corr"] == want["num_corr"] and frob(got["T"], want["T"]) < 1e-5, frob(got["T"], want["T"])


# ---- degenerate geometry -----------------------------------------------------------------------------------------
T_SMALL = synth.rigid_from_axis_angle([1, 1, 1], 0.01, [0.003, -0.002, 0.001])


def _sheet(n, seed, thickness=0.0, corridor=False):
    """Points on z = 0 over [0,1)^2 (uniform thickness in z, optionally a second plane at z = 0.3: a corridor), with
    surface normals +z (floor) / -z (ceiling)."""
    rng = np.random.default_rng(seed)
    xy = rng.random((n, 2))
    u = rng.random(n) - 0.5
    top = (rng.random(n) < 0.5) if corridor else np.zeros(n, bool)
    z = thickness * u + 0.3 * top
    pts = np.stack([xy[:, 0], xy[:, 1], z], 1).astype(np.float32)
    nrm = np.zeros((n, 3), np.float32)
    nrm[:, 2] = np.where(top, -1.0, 1.0)
    return pts, nrm


def _thickness_for_ratio(n, seed, target):
    """Thickness at which the covariance of _sheet(n, seed) has det / |.|_F^3 = target (bisection; det grows with
    the thickness squared)."""
    lo, hi = 0.0, 0.1
    for _ in range(80):
        mid = 0.5 * (lo + hi)
        p, _ = _sheet(n, seed, mid)
        C = np.cov(p.astype(np.float64).T, bias=True)
        lo, hi = (mid, hi) if icp_ref.det_ratio(C) < target else (lo, mid)
    return 0.5 * (lo + hi)


def _run_both_loops(cb, ctx, dst, nrm, src, src_n, T0, max_d2, metric, kw, iters):
    icp = cb.Icp(ctx, cb.Cloud(ctx, dst, nrm), cb.Cloud(ctx, src, src_n))
    out = {}
    for host_loop in (False, True):
        out[host_loop] = icp.estimate(metric=metric, max_iter=iters, tol=0.0, max_d2=max_d2, T_init=T0,
                                      host_loop=host_loop, **kw)
    return icp, out


@pytest.mark.parametrize("case", ["plane", "thin_below", "thin_above", "corridor"])
def test_p2p_on_planar_scenes(cb, ctx, orc, case):
    """sigma of a plane has rank 2 (the SVD path, u2 = u0 x u1; the Kabsch rotation is still unique); a thin slab
    lands on either side of the polar iteration's acceptance threshold; a corridor is well conditioned. One step
    against the float64 reference in both loops, then five iterations: loops agree, and agree with the oracle."""
    n, seed = 3000, 50
    thick = {"plane": 0.0, "corridor": 0.0, "thin_below": _thickness_for_ratio(n, seed, 1e-6 * (1 - 1e-2)),
             "thin_above": _thickness_for_ratio(n, seed, 1e-6 * (1 + 1e-2))}[case]
    dst, nrm = _sheet(n, seed, thick, corridor=case == "corridor")
    src = synth.apply(synth.invert(T_SMALL), dst)
    # thin slabs: start next to the truth so that every point is matched to itself and sigma ~ the slab's covariance
    T0 = (synth.rigid_from_axis_angle([0, 0, 1], 1e-3, [0, 0, 0]) @ np.vstack([T_SMALL, [0, 0, 0, 1]])
          if case.startswith("thin") else np.hstack([np.eye(3), np.zeros((3, 1))])).astype(np.float32)
    max_d2 = np.float32(0.02**2)
    icp, one = _run_both_loops(cb, ctx, dst, None, src, None, T0, max_d2, "p2p", {}, 1)
    f, s = _pairs(cb, orc, icp, dst, src, T0, max_d2, {})
    Tr, info = icp_ref.p2p_step(dst, src, T0, f, s)
    want_polar = {"plane": False, "thin_below": False, "thin_above": True, "corridor": True}[case]
    assert info["polar"] == want_polar, (case, icp_ref.det_ratio(info["sigma"]))
    if case == "plane":
        assert np.linalg.matrix_rank(info["sigma"], tol=1e-12) == 2
    for host_loop, r in one.items():
        assert r["num_corr"] == len(f)
        assert frob(r["T"], Tr) < 1e-6, (case, host_loop, frob(r["T"], Tr))
    _, five = _run_both_loops(cb, ctx, dst, None, src, None, T0, max_d2, "p2p", {}, 5)
    assert five[True]["num_corr"] == five[False]["num_corr"] and frob(five[True]["T"], five[False]["T"]) < 1e-6
    want = orc.icp(dst, src, orc.BruteKnn(dst), metric="p2p", max_iter=5, tol=0.0, max_d2=max_d2, T_init=T0)
    assert five[False]["num_corr"] == want["num_corr"] and frob(five[False]["T"], want["T"]) < 1e-5


@pytest.mark.parametrize("case", ["line", "coincident"])
def test_p2p_rank_deficient_rotation_is_proper_and_maps_the_pairs(cb, ctx, orc, case):
    """A pole (rank-1 sigma) and a cloud of coincident points (sigma = 0): the rotation is not unique, but both loops
    must return a proper rotation that maps every matched source point onto its destination."""
    rng = np.random.default_rng(51)
    n = 2000
    if case == "line":
        dst = np.zeros((n, 3), np.float32)
        dst[:, 0] = rng.random(n)
    else:
        dst = np.tile(np.float32([[0.3, 0.6, 0.2]]), (n, 1))
    src = synth.apply(synth.invert(T_SMALL), dst)
    T0 = T_SMALL.astype(np.float32)
    max_d2 = np.float32(0.01**2)
    icp, one = _run_both_loops(cb, ctx, dst, None, src, None, T0, max_d2, "p2p", {}, 1)
    f, s = _pairs(cb, orc, icp, dst, src, T0, max_d2, {})
    _, info = icp_ref.p2p_step(dst, src, T0, f, s)
    assert not info["polar"] and np.linalg.matrix_rank(info["sigma"], tol=1e-9) == (1 if case == "line" else 0)
    for host_loop, r in one.items():
        assert r["num_corr"] == len(f) == n
        assert _proper(r["T"]), (case, host_loop)
        err = np.abs(icp_ref.apply(r["T"], src[s]) - dst[f]).max()
        assert err < 2e-5, (case, host_loop, err)
        if case == "coincident":  # sigma = 0: the SVD of zero is the identity, the update a translation
            assert np.abs(r["T"][:, :3] - T0[:, :3]).max() < 1e-6


@pytest.mark.parametrize("case", ["plane", "corridor"])
@pytest.mark.parametrize("symmetric", [False, True])
def test_combined_metric_on_planar_scenes(cb, ctx, orc, case, symmetric):
    """Point-to-plane with surface normals on a plane / corridor: AtA is (nearly) rank 3 (rotation about z and the
    in-plane translation are unconstrained by the plane terms), made solvable by a small point-to-point weight. The
    float64 reference reports the condition number; the tolerance scales with it."""
    dst, nrm = _sheet(3000, 52, corridor=case == "corridor")
    src = synth.apply(synth.invert(T_SMALL), dst)
    src_n = (nrm.astype(np.float64) @ synth.invert(T_SMALL)[:, :3].T).astype(np.float32) if symmetric else None
    T0 = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)
    max_d2 = np.float32(0.02**2)
    kw = dict(w_pt=1e-3, w_pl=1.0)
    icp, one = _run_both_loops(cb, ctx, dst, nrm, src, src_n, T0, max_d2, "combined", kw, 1)
    f, s = _pairs(cb, orc, icp, dst, src, T0, max_d2, {})
    Tr, info = _ref_step(dst, src, T0, f, s, "combined", kw, dst_n=nrm, src_n=src_n)
    cond = info["cond"]
    assert cond > 1e3, cond  # the case is what it claims to be
    x = np.linalg.solve(info["A"], info["b"])
    # fp32 inputs of the normal equations (d, s, v, e are rounded to float on the device): |dx| ~ eps_32 cond |x|
    tol = 1e-6 + 16 * np.finfo(np.float32).eps * cond * np.abs(x).max()
    for host_loop, r in one.items():
        assert r["num_corr"] == len(f)
        assert _proper(r["T"]) and frob(r["T"], Tr) < tol, (case, host_loop, frob(r["T"], Tr), tol, cond)
    _, five = _run_both_loops(cb, ctx, dst, nrm, src, src_n, T0, max_d2, "combined", kw, 5)
    assert five[True]["num_corr"] == five[False]["num_corr"]
    assert frob(five[True]["T"], five[False]["T"]) < tol, (frob(five[True]["T"], five[False]["T"]), tol)
    print(f"\n{case} symmetric={symmetric}: cond(AtA) = {cond:.2e}, one step |T - T_ref64| = "
          f"{max(frob(r['T'], Tr) for r in one.values()):.2e} (tol {tol:.1e})")


# ---- sizes at block and reduction-group boundaries --------------------------------------------------------------
@pytest.mark.parametrize("n_dst", [1, 2])
@pytest.mark.parametrize("n_src", [1, 2, 3, 255, 256, 257, 16384, 16385, 32769])
def test_sizes_at_block_and_group_boundaries(cb, ctx, orc, n_src, n_dst):
    """256-thread blocks reduced in groups of 64 (kReduceGroup): 16385 and 32769 sources leave a last group of one
    block. One or two destination points: sigma = 0 (translation only) or rank 1; one and two sources are the 1- and
    2-correspondence cases of kabsch_from_moments."""
    rng = np.random.default_rng(n_src * 10 + n_dst)
    dst = np.float32([[0.2, 0.3, 0.4], [0.7, 0.3, 0.4]])[:n_dst]
    src = (dst[rng.integers(0, n_dst, n_src)] + (rng.random((n_src, 3)) - 0.5) * 0.02).astype(np.float32)
    max_d2 = np.float32(0.05**2)
    T0 = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)
    icp, one = _run_both_loops(cb, ctx, dst, None, src, None, T0, max_d2, "p2p", {}, 1)
    f, s = _pairs(cb, orc, icp, dst, src, T0, max_d2, {})
    assert len(f) == n_src
    Tr, info = icp_ref.p2p_step(dst, src, T0, f, s)
    assert not info["polar"]
    for host_loop, r in one.items():
        assert r["num_corr"] == n_src and _proper(r["T"]), host_loop
        if n_dst == 1 or n_src == 1:  # sigma = 0: R = I, t = mu_d - mu_q, unique
            assert frob(r["T"], Tr) < 1e-6, (host_loop, frob(r["T"], Tr))
        else:  # rank 1: R v0 = u0 and t = mu_d - R mu_q
            U, _, Vt = np.linalg.svd(info["sigma"])
            R = r["T"][:, :3].astype(np.float64)
            assert np.abs(R @ Vt[0] - U[:, 0]).max() < 1e-5, host_loop
            mud, muq = dst[f].astype(np.float64).mean(0), src[s].astype(np.float64).mean(0)
            assert np.abs(r["T"][:, 3] - (mud - R @ muq)).max() < 1e-5, host_loop
    if n_dst == 1:
        # a few iterations: the first translation centres the source on the point, after which the update is the
        # identity. (The oracle is no yardstick here: its fp32 sigma of a single destination point is rounding noise,
        # and so is the rotation the SVD makes of it.)
        _, three = _run_both_loops(cb, ctx, dst, None, src, None, T0, max_d2, "p2p", {}, 3)
        for r in three.values():
            assert r["num_corr"] == n_src and frob(r["T"], Tr) < 1e-6, frob(r["T"], Tr)
    # no correspondence at all: identity, count 0 (transform_estimation.hpp:20-23)
    far = (src + np.float32(5.0)).astype(np.float32)
    _, none = _run_both_loops(cb, ctx, dst, None, far, None, T0, max_d2, "p2p", {}, 1)
    for r in none.values():
        assert r["num_corr"] == 0 and np.array_equal(r["T"], T0)
