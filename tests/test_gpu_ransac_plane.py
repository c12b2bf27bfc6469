"""GPU parity of plane RANSAC (cb_plane_score, cb_plane_residuals, cb_ransac_plane) against the oracle
(oracle/plane_ransac_oracle.cpp) and numpy, and device-versus-host bit identity of the hypothesis fit (plane_fit.hpp)."""
import os

import numpy as np
import pytest

import cxx
from cilantro_b200 import synth
from oracle import ransac_plane as orp
from test_oracle_ransac_plane import fit_cases, np_residuals, same_bits

pytestmark = pytest.mark.gpu

F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
THRESHOLDS = [0.0, 1e-30, 0.01, np.inf, -1.0, np.nan]


def random_planes(pts, H, seed):
    samples, planes = orp.hypotheses(pts, seed, H)
    return planes


# ---- cb_plane_score ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [1, 255, 256, 257, 1024, 1025, 2500])
def test_plane_score_counts_bitexact_batch_sizes(cb, ctx, H):
    pts = synth.plane_scene(30000, seed=2)["points"]
    planes = random_planes(pts, H, seed=H)
    got = cb.plane_score(ctx, cb.Cloud(ctx, pts), planes, 0.01)
    assert np.array_equal(got, orp.score(pts, planes, 0.01))


@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 256, 257, 2047, 2048, 2049, 65536, 65537])
@pytest.mark.parametrize("thresh", THRESHOLDS)
def test_plane_score_counts_bitexact_tile_boundaries(cb, ctx, n, thresh):
    rng = np.random.default_rng(n)
    pts = rng.normal(size=(n, 3)).astype(F32)
    pts[::3, 2] = 0.0
    if n > 10:
        pts[3] = [np.nan, 0, 0]
        pts[4] = [np.inf, 0, 0]
    planes = np.vstack([[0, 0, 1, 0], random_planes(pts, 40, seed=1), np.full((1, 4), np.nan)]).astype(F32)
    got = cb.plane_score(ctx, cb.Cloud(ctx, pts), planes, thresh)
    assert np.array_equal(got, orp.score(pts, planes, thresh))


# ---- cb_plane_residuals ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("thresh", THRESHOLDS)
def test_plane_residuals_bits_and_inlier_list(cb, ctx, thresh):
    sc = synth.plane_scene(70001, seed=4)
    pts = sc["points"].copy()
    pts[10] = [np.nan, 1, 1]
    pts[11] = [np.inf, 1, 1]
    cloud = cb.Cloud(ctx, pts)
    for plane in (sc["planes"][0].astype(F32), random_planes(pts, 1, 3)[0]):
        res, inl = cb.plane_residuals(ctx, cloud, plane, thresh)
        want = np_residuals(pts, plane)
        assert same_bits(res, want)
        assert np.array_equal(inl, np.nonzero(want <= F32(thresh))[0])
        assert np.all(np.diff(inl) > 0)


# ---- cb_ransac_plane ---------------------------------------------------------------------------------------------------
def check_no_reestimate(got, want):
    assert (got["iterations"], got["best_iteration"]) == (want["iterations"], want["best_iteration"])
    assert same_bits(got["hyp_plane"], want["hyp_plane"]) and same_bits(got["plane"], want["plane"])
    assert got["num_inliers"] == want["num_inliers"] and np.array_equal(got["inliers"], want["inliers"])
    assert same_bits(got["residuals"], want["residuals"])


def angle(a, b):
    a, b = np.asarray(a[:3], np.float64), np.asarray(b[:3], np.float64)
    c = abs(float(a @ b)) / (np.linalg.norm(a) * np.linalg.norm(b))
    return float(np.arccos(min(1.0, c)))


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
@pytest.mark.parametrize("scene_seed", [5, 6])
def test_ransac_plane_matches_oracle(cb, ctx, seed, scene_seed):
    sc = synth.plane_scene(40000, seed=scene_seed)
    pts = sc["points"]
    cloud = cb.Cloud(ctx, pts)
    kw = dict(max_iter=250, thresh=0.01, inlier_count_thresh=int(0.15 * pts.shape[0]))
    got = cb.ransac_plane(ctx, cloud, seed, re_estimate=False, **kw)
    check_no_reestimate(got, orp.ransac_plane(pts, seed, re_estimate=False, **kw))
    got = cb.ransac_plane(ctx, cloud, seed, **kw)
    want = orp.ransac_plane(pts, seed, accum_double=True, **kw)
    assert (got["iterations"], got["best_iteration"]) == (want["iterations"], want["best_iteration"])
    assert same_bits(got["hyp_plane"], want["hyp_plane"])
    assert angle(got["plane"], want["plane"]) < 1e-5
    assert abs(got["num_inliers"] - want["num_inliers"]) <= 3
    _, inl = cb.plane_residuals(ctx, cloud, got["plane"], 0.01)
    assert np.array_equal(got["inliers"], inl)


def test_ransac_plane_finds_the_floor(cb, ctx):
    sc = synth.plane_scene(200000, seed=9)
    pts = sc["points"]
    got = cb.ransac_plane(ctx, cb.Cloud(ctx, pts), 3, max_iter=250, thresh=0.01,
                          inlier_count_thresh=int(0.4 * pts.shape[0]))
    floor = sc["planes"][0]
    assert angle(got["plane"], floor) < 2e-3
    r = np.abs(pts.astype(np.float64) @ floor[:3] + floor[3])
    labelled = int((sc["labels"] == 0).sum())
    in_slab = int((r <= 0.01).sum())  # the floor plus the clutter inside its slab
    assert abs(got["num_inliers"] - labelled) <= 0.02 * labelled
    assert got["num_inliers"] <= in_slab * 1.02


def test_reference_example_recipe_and_no_early_exit(cb, ctx):
    sc = synth.plane_scene(100000, seed=12)
    pts = sc["points"]
    cloud = cb.Cloud(ctx, pts)
    kw = dict(max_iter=250, thresh=0.01, inlier_count_thresh=int(0.15 * pts.shape[0]))  # examples/ransac_plane_estimator.cpp
    got = cb.ransac_plane(ctx, cloud, 21, **kw)
    want = orp.ransac_plane(pts, 21, accum_double=True, **kw)
    assert got["iterations"] < 250 and got["iterations"] == want["iterations"]
    kw["inlier_count_thresh"] = pts.shape[0] + 1  # unreachable: every iteration runs
    got = cb.ransac_plane(ctx, cloud, 21, re_estimate=False, **kw)
    want = orp.ransac_plane(pts, 21, re_estimate=False, **kw)
    assert got["iterations"] == 250
    check_no_reestimate(got, want)


def plane_contains(plane, pts, tol):
    pl = np.asarray(plane, np.float64)
    return np.isfinite(pl).all() and abs(np.linalg.norm(pl[:3]) - 1) < 1e-5 and \
        np.abs(np.asarray(pts, np.float64) @ pl[:3] + pl[3]).max() <= tol


@pytest.mark.parametrize("n", [0, 1, 2, 3])
@pytest.mark.parametrize("re_estimate", [False, True])
def test_tiny_clouds(cb, ctx, n, re_estimate):
    pts = np.array([[0.5, 0.25, 1.0], [2.0, -1.0, 1.5], [0.0, 3.0, -2.0]], F32)[:n]
    kw = dict(max_iter=7, thresh=0.01, re_estimate=re_estimate)
    got = cb.ransac_plane(ctx, cb.Cloud(ctx, pts), 5, **kw)
    want = orp.ransac_plane(pts, 5, accum_double=True, **kw)
    assert (got["iterations"], got["best_iteration"], got["num_inliers"]) == \
        (want["iterations"], want["best_iteration"], want["num_inliers"])
    assert same_bits(got["hyp_plane"], want["hyp_plane"])
    assert np.array_equal(got["inliers"], want["inliers"])
    if n < 2:
        assert np.isnan(got["plane"]).all() and got["num_inliers"] == 0
    else:
        assert plane_contains(got["plane"], pts, 1e-5)


@pytest.mark.parametrize("kind", ["collinear", "grid", "duplicates"])
def test_degenerate_clouds(cb, ctx, kind):
    rng = np.random.default_rng(3)
    if kind == "collinear":
        t = rng.integers(-50, 50, 3000).astype(F32)
        pts = np.column_stack([t, 2 * t + 1, -t]).astype(F32)
    elif kind == "grid":
        g = np.arange(12, dtype=F32)
        pts = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    else:
        base = rng.normal(size=(40, 3)).astype(F32)
        pts = base[rng.integers(0, 40, 5000)]
    cloud = cb.Cloud(ctx, pts)
    kw = dict(max_iter=60, thresh=0.01, inlier_count_thresh=pts.shape[0])
    got = cb.ransac_plane(ctx, cloud, 8, re_estimate=False, **kw)
    check_no_reestimate(got, orp.ransac_plane(pts, 8, re_estimate=False, **kw))
    got = cb.ransac_plane(ctx, cloud, 8, **kw)
    want = orp.ransac_plane(pts, 8, accum_double=True, **kw)
    assert (got["iterations"], got["best_iteration"]) == (want["iterations"], want["best_iteration"])
    hyp_inl = orp.residuals(pts, want["hyp_plane"], 0.01)[1]
    if kind == "collinear":  # rank-deficient re-estimation: any plane through the line is an answer
        assert plane_contains(got["plane"], pts[hyp_inl], 1e-3)
    else:
        assert angle(got["plane"], want["plane"]) < 1e-5
        assert abs(got["num_inliers"] - want["num_inliers"]) <= 3


def test_non_finite_rows_never_inliers_nor_poison(cb, ctx):
    sc = synth.plane_scene(50000, seed=14)
    pts = sc["points"].copy()
    bad = np.arange(0, 50000, 97)
    pts[bad[0::3]] = np.nan
    pts[bad[1::3], 1] = np.inf
    pts[bad[2::3], 2] = -np.inf
    cloud = cb.Cloud(ctx, pts)
    kw = dict(max_iter=250, thresh=0.01, inlier_count_thresh=int(0.4 * pts.shape[0]))
    got = cb.ransac_plane(ctx, cloud, 2, re_estimate=False, **kw)
    check_no_reestimate(got, orp.ransac_plane(pts, 2, re_estimate=False, **kw))
    got = cb.ransac_plane(ctx, cloud, 2, **kw)
    want = orp.ransac_plane(pts, 2, accum_double=True, **kw)
    assert np.isfinite(got["plane"]).all()
    assert angle(got["plane"], want["plane"]) < 1e-5
    assert not np.isin(got["inliers"], bad).any()


def test_rejected_inputs(cb, ctx):
    pts = synth.plane_scene(1000, seed=1)["points"]
    with pytest.raises(cb.CbError):
        cb.ransac_plane(ctx, cb.Cloud(ctx, pts, index_offset=5), 1)


# ---- the fit header: device build == host build ----------------------------------------------------------------------
def test_fit_device_bits_equal_host_bits(tmp_path):
    src = os.path.join(ROOT, "tests", "cuda", "plane_fit_harness.cu")
    inc = ["-I" + cxx.CSRC]
    exe_d = cxx.harness(src, str(tmp_path / "fit_dev"), inc, device=True)
    exe_h = cxx.harness(src, str(tmp_path / "fit_host"), inc, device=False)
    rng = np.random.default_rng(17)
    cases = fit_cases() + [rng.normal(size=(3, 3)) * 10.0 ** rng.integers(-20, 20) for _ in range(2000)]
    rec = np.zeros((len(cases), 10), F32)
    for i, s in enumerate(cases):
        s = np.asarray(s, F32).reshape(-1, 3)
        rec[i, :s.size] = s.reshape(-1)
        rec[i, 9] = s.shape[0]
    rec.tofile(tmp_path / "in.bin")
    outs = []
    for exe in (exe_d, exe_h):
        cxx.run(exe, tmp_path / "in.bin", tmp_path / "out.bin")
        outs.append(np.fromfile(tmp_path / "out.bin", F32).reshape(-1, 4))
    assert same_bits(outs[0], outs[1])
    for i, s in enumerate(cases):  # and both are the oracle's (and numpy's, test_oracle_ransac_plane.py) closed form
        assert same_bits(outs[0][i], orp.fit(np.asarray(s, F32)))
