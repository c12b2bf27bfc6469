"""The device ICP loop's cached pass reading packed 12-byte coordinates (icp_loop.cu, icp_cached_pipe_kernel): each warp
streams its 32 queries as one 384-byte window of packed source xyz that 24 lanes copy and every lane reads from, and
gathers each cached match (and its normal) as three 4-byte copies from packed destination xyz.

Each case runs the loop for 1, 2 and 5 iterations and checks that the cache names the brute-force nearest neighbour of
every query (of a sample at 10^6 queries) at the transform the last search used, that the device loop's transform and
correspondence count are bit-identical to the host-driven loop's, and that a second run is byte-identical.
"""
import numpy as np
import pytest

from cilantro_b200 import synth

pytestmark = pytest.mark.gpu

TILE_P2P = 256  # queries per tile of the p2p pass


def _rigid(angle, t):
    return synth.rigid_from_axis_angle([1, 2, 3], angle, t)


def _check_cache(orc, dst, icp, src, max_d2, rows=None):
    T_search, near, searched = icp.loop_cache()
    if rows is not None:
        src, near = src[rows], near[rows]
    idx, d2 = orc.BruteKnn(dst).query(orc.transform_points(T_search, src), np.float32(3.0e38))
    inside = d2 < max_d2
    assert np.array_equal(near[inside], idx[inside])
    named = (~inside) & (near >= 0)
    assert np.array_equal(near[named], idx[named])
    return searched


def _run(cb, ctx, orc, dst, src, max_d2, dst_nrm=None, src_nrm=None, rows=None, iters_list=(1, 2, 5), **kw):
    """Returns the searched count of the last iteration of each run."""
    searched = []
    for iters in iters_list:
        out = []
        for _ in range(2):
            icp = cb.Icp(ctx, cb.Cloud(ctx, dst, dst_nrm), cb.Cloud(ctx, src, src_nrm))
            r = icp.estimate(tol=0.0, timing=0, max_iter=iters, max_d2=max_d2, host_loop=False, **kw)
            out.append((icp, r))
        (icp, a), (_, b) = out
        assert a["iterations"] == b["iterations"] == iters
        assert a["num_corr"] == b["num_corr"]
        assert a["T"].tobytes() == b["T"].tobytes()
        searched.append(_check_cache(orc, dst, icp, src, max_d2, rows))
        h = icp.estimate(tol=0.0, timing=0, max_iter=iters, max_d2=max_d2, host_loop=True, **kw)
        assert h["iterations"] == iters and h["num_corr"] == a["num_corr"], (iters, h["num_corr"], a["num_corr"])
        assert h["T"].tobytes() == a["T"].tobytes(), iters
    return searched


@pytest.mark.parametrize("n_src", [1, 31, 33, 255, 257, 32 * 411 + 17, TILE_P2P * 37 + 13])
def test_window_and_tile_edges(cb, ctx, orc, n_src):
    """n_src inside the first window, one short of a window, one past it, around one tile, and ending mid-window. With
    n_src of a few thousand at most the grid has more resident blocks than there are tiles."""
    dst, src, _, _ = synth.icp_pair(30000, seed=41, noise=0.002, n_src=n_src, T_ref=_rigid(0.03, [0.01, 0.004, -0.006]))
    _run(cb, ctx, orc, dst, src, np.float32(0.05**2), metric="p2p")


def test_million_and_three(cb, ctx, orc):
    """1 000 003 queries: several tiles per block and a last window of 3 queries. The cache is checked on the first and
    last 3 000 queries and on a random sample."""
    n = 1_000_003
    dst, src, _, _ = synth.icp_pair(200_000, seed=42, noise=0.002, n_src=n, T_ref=_rigid(0.02, [0.005, -0.004, 0.006]))
    rng = np.random.default_rng(9)
    rows = np.unique(np.concatenate([np.arange(3000), np.arange(n - 3000, n), rng.integers(0, n, 6000)]))
    _run(cb, ctx, orc, dst, src, np.float32(0.05**2), rows=rows, iters_list=(2, 5), metric="p2p")


def test_almost_every_query_flagged(cb, ctx, orc):
    """A large first step: the warm iterations flag nearly every query, so every lane's window is read and every warp's
    list is full."""
    n = 40000
    dst, src, _, _ = synth.icp_pair(n, seed=43, noise=0.001, T_ref=_rigid(0.15, [0.12, -0.08, 0.1]))
    searched = _run(cb, ctx, orc, dst, src, np.float32(0.3**2), iters_list=(2, 3), metric="p2p")
    assert searched[0] > n // 2, searched


def test_every_destination_point_matched(cb, ctx, orc):
    """A noise-free source displaced far less than the point spacing: every destination point is some query's match,
    so the last point of the cell-sorted destination is gathered too, from the last 12 bytes of its packed copy."""
    n = 20000
    dst, src, _, _ = synth.icp_pair(n, seed=44, noise=0.0, T_ref=_rigid(0.002, [0.0004, 0.0002, -0.0003]))
    _run(cb, ctx, orc, dst, src, np.float32(0.05**2), metric="p2p")
    icp = cb.Icp(ctx, cb.Cloud(ctx, dst), cb.Cloud(ctx, src))
    icp.estimate(tol=0.0, timing=0, max_iter=3, max_d2=np.float32(0.05**2), metric="p2p")
    _, near, _ = icp.loop_cache()
    assert np.unique(near).size == n and near.min() >= 0


@pytest.mark.parametrize("src_normals", [False, True])
def test_combined_metric(cb, ctx, orc, src_normals):
    """The combined pass (two queries per thread, two windows per warp and tile, normals gathered from the packed copy),
    with and without source normals (the symmetric plane term)."""
    n = 50000
    dst, src, nrm, _ = synth.icp_pair(n, seed=45, noise=0.002, with_normals=True, n_src=n - 45,
                                      T_ref=_rigid(0.04, [0.02, -0.01, 0.015]))
    src_nrm = None
    if src_normals:
        v = np.random.default_rng(6).normal(size=src.shape)
        src_nrm = (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)
    _run(cb, ctx, orc, dst, src, np.float32(0.05**2), nrm, src_nrm, metric="combined", w_pt=0.1, w_pl=1.0)
