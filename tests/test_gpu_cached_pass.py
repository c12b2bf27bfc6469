"""The device ICP loop's cached pass (icp_loop.cu, icp_cached_pipe_kernel) at the edges of its per-warp lists of
flagged queries and of its tiling: every warp searches the queries it flagged after its last tile, from a list in
global memory, in the shared memory its pipeline used.

Each case runs the loop for a few iterations and checks that the cache names the brute-force nearest neighbour of
every query at the transform the last search used, and that a second run gives a byte-identical transform.
"""
import numpy as np
import pytest

from cilantro_b200 import synth

pytestmark = pytest.mark.gpu

TILE_P2P = 256  # queries per tile of the p2p pass (pipe_qpt(false) x kBlock)


def _rigid(angle, t):
    return synth.rigid_from_axis_angle([1, 2, 3], angle, t)


def _check_cache(orc, dst, icp, src, max_d2):
    T_search, near, searched = icp.loop_cache()
    idx, d2 = orc.BruteKnn(dst).query(orc.transform_points(T_search, src), np.float32(3.0e38))
    inside = d2 < max_d2
    assert np.array_equal(near[inside], idx[inside])
    named = (~inside) & (near >= 0)
    assert np.array_equal(near[named], idx[named])
    return searched


def _run_twice(cb, ctx, dst, src, dst_nrm=None, src_nrm=None, **kw):
    out = []
    for _ in range(2):
        icp = cb.Icp(ctx, cb.Cloud(ctx, dst, dst_nrm), cb.Cloud(ctx, src, src_nrm))
        r = icp.estimate(tol=0.0, timing=0, **kw)
        out.append((icp, r))
    (icp, a), (_, b) = out
    assert a["iterations"] == b["iterations"] == kw["max_iter"]
    assert a["num_corr"] == b["num_corr"]
    assert a["T"].tobytes() == b["T"].tobytes()
    return icp, a


@pytest.mark.parametrize("iters", [2, 3])
def test_every_query_flagged_after_a_large_first_step(cb, ctx, orc, iters):
    """A source far off its destination: the first update moves every query by more than its exclusion radius, so the
    warm iterations flag (nearly) every query and every warp's list is full."""
    n = 40000
    dst, src, _, _ = synth.icp_pair(n, seed=31, noise=0.001, T_ref=_rigid(0.15, [0.12, -0.08, 0.1]))
    max_d2 = np.float32(0.3**2)
    icp, _ = _run_twice(cb, ctx, dst, src, metric="p2p", max_iter=iters, max_d2=max_d2)
    searched = _check_cache(orc, dst, icp, src, max_d2)
    assert searched > n // 2, searched


@pytest.mark.parametrize("n_src", [TILE_P2P * 37 + 13, TILE_P2P - 57, 31, 20000])
def test_tile_and_grid_edges(cb, ctx, orc, n_src):
    """n_src not a multiple of the tile, smaller than one tile, than one warp, and fewer tiles than
    the resident blocks of the grid."""
    dst, src, _, _ = synth.icp_pair(30000, seed=7, noise=0.002, n_src=n_src, T_ref=_rigid(0.03, [0.01, 0.004, -0.006]))
    max_d2 = np.float32(0.05**2)
    for iters in (1, 2, 5):
        icp, _ = _run_twice(cb, ctx, dst, src, metric="p2p", max_iter=iters, max_d2=max_d2)
        _check_cache(orc, dst, icp, src, max_d2)


@pytest.mark.parametrize("src_normals", [False, True])
def test_combined_metric(cb, ctx, orc, src_normals):
    """The combined pass (two queries per thread, normals gathered in stage B), with and without source normals (the
    symmetric plane term)."""
    n = 50000
    dst, src, nrm, _ = synth.icp_pair(n, seed=12, noise=0.002, with_normals=True, n_src=n - 333,
                                      T_ref=_rigid(0.04, [0.02, -0.01, 0.015]))
    src_nrm = None
    if src_normals:
        v = np.random.default_rng(3).normal(size=src.shape)
        src_nrm = (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)
    max_d2 = np.float32(0.05**2)
    for iters in (2, 5):
        icp, _ = _run_twice(cb, ctx, dst, src, nrm, src_nrm, metric="combined", w_pt=0.1, w_pl=1.0, max_iter=iters,
                            max_d2=max_d2)
        _check_cache(orc, dst, icp, src, max_d2)


def test_survey_pose_before_and_after_the_hand_over(cb, ctx, orc):
    """SURVEY 8d's pose on a dense cloud: a large share of the queries is flagged in every warm iteration. The first
    batch stays on the device loop (exact cache, deterministic); a longer run is handed over to the host loop and
    matches the host loop alone."""
    n = 200000
    dst, src, _, _ = synth.icp_pair(n, seed=4, noise=0.001, T_ref=synth.t_ref_default())
    max_d2 = np.float32(0.02**2)
    icp, _ = _run_twice(cb, ctx, dst, src, metric="p2p", max_iter=4, max_d2=max_d2)
    searched = _check_cache(orc, dst, icp, src, max_d2)
    assert searched > n // 50, searched
    kw = dict(metric="p2p", max_iter=9, tol=0.0, max_d2=max_d2)
    a = icp.estimate(host_loop=True, **kw)
    b = icp.estimate(host_loop=False, **kw)
    c = icp.estimate(host_loop=False, **kw)
    assert a["iterations"] == b["iterations"] == 9 and a["num_corr"] == b["num_corr"] == c["num_corr"]
    assert np.linalg.norm(a["T"].astype(np.float64) - b["T"]) < 1e-6
    assert b["T"].tobytes() == c["T"].tobytes()
