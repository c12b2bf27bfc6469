"""The device ICP loop's cold pass (icp_loop.cu, icp_search_kernel): the first iteration of a call, where a
persistent grid of warps walks the 32-query chunks of the source round-robin and searches every query.

Each case runs the loop for 1, 2 and 5 iterations, checks that the cache names the brute-force nearest neighbour of
every query at the transform the last search used, and that a second run gives a byte-identical transform.
"""
import numpy as np
import pytest

from cilantro_b200 import synth

pytestmark = pytest.mark.gpu


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


def _run(cb, ctx, orc, dst, src, max_d2, dst_nrm=None, src_nrm=None, **kw):
    for iters in (1, 2, 5):
        out = []
        for _ in range(2):
            icp = cb.Icp(ctx, cb.Cloud(ctx, dst, dst_nrm), cb.Cloud(ctx, src, src_nrm))
            r = icp.estimate(tol=0.0, timing=0, max_iter=iters, max_d2=max_d2, **kw)
            out.append((icp, r))
        (icp, a), (_, b) = out
        assert a["iterations"] == b["iterations"] == iters
        assert a["num_corr"] == b["num_corr"]
        assert a["T"].tobytes() == b["T"].tobytes()
        searched = _check_cache(orc, dst, icp, src, max_d2)
        if iters == 1:
            assert searched == src.shape[0]


@pytest.mark.parametrize("n_src", [256 * 37 + 13, 20, 5000, 150001])
def test_chunk_and_grid_edges(cb, ctx, orc, n_src):
    """n_src not a multiple of 32 or 256, below one warp, fewer chunks than the grid has warps, and several chunks
    per warp."""
    dst, src, _, _ = synth.icp_pair(60000, seed=21, noise=0.002, n_src=n_src, T_ref=_rigid(0.03, [0.01, 0.004, -0.006]))
    _run(cb, ctx, orc, dst, src, np.float32(0.05**2), metric="p2p")


def test_queries_outside_the_grid(cb, ctx, orc):
    """An initial pose that puts a large share of the queries outside the destination grid (the exact fallback)."""
    dst, src, _, _ = synth.icp_pair(30000, seed=22, noise=0.002)
    T_init = _rigid(0.0, [0.45, -0.3, 0.2]).astype(np.float32)
    _run(cb, ctx, orc, dst, src, np.float32(0.5**2), metric="p2p", T_init=T_init)


def test_duplicated_points(cb, ctx, orc):
    """Destination points repeated exactly and queries on them: exact ties, resolved on the lowest index."""
    dst, src, _, _ = synth.icp_pair(20000, seed=23, noise=0.002)
    dst = np.concatenate([dst, dst[:5000], dst[:2000]])
    src = np.concatenate([src[:15000], dst[:3000]])
    _run(cb, ctx, orc, dst, src, np.float32(0.05**2), metric="p2p")


def test_tiny_radius(cb, ctx, orc):
    """max_d2 far below the spacing: almost no correspondence, every cache entry decided by the radius."""
    dst, src, _, _ = synth.icp_pair(30000, seed=24, noise=0.002)
    _run(cb, ctx, orc, dst, src, np.float32(1e-4**2), metric="p2p")


def test_large_rotation(cb, ctx, orc):
    """A 2.5 rad initial rotation: the 32 queries of a chunk are far apart in the destination grid."""
    dst, src, _, _ = synth.icp_pair(40000, seed=25, noise=0.002)
    c = np.array([0.5, 0.5, 0.5])
    T_init = _rigid(2.5, [0, 0, 0])
    T_init[:, 3] = c - T_init[:, :3] @ c
    _run(cb, ctx, orc, dst, src, np.float32(0.1**2), metric="p2p", T_init=T_init.astype(np.float32))


@pytest.mark.parametrize("src_normals", [False, True])
def test_combined_metric(cb, ctx, orc, src_normals):
    """The combined metric's cold pass (its own register budget), with and without source normals."""
    n = 50000
    dst, src, nrm, _ = synth.icp_pair(n, seed=26, noise=0.002, with_normals=True, n_src=n - 77,
                                      T_ref=_rigid(0.04, [0.02, -0.01, 0.015]))
    src_nrm = None
    if src_normals:
        v = np.random.default_rng(5).normal(size=src.shape)
        src_nrm = (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)
    _run(cb, ctx, orc, dst, src, np.float32(0.05**2), nrm, src_nrm, metric="combined", w_pt=0.1, w_pl=1.0)
