"""The device ICP loop's cache after 1, 2 and 5 iterations on clouds that stress the pooled region scan of the wide
grid search (warp_search_wide.cuh; one lane per region in the cold search, lane pairs in the cached pass): crowded
cells whose regions hold many points, empty rows, lattices with exact 2-, 4- and 8-way ties, queries outside the grid,
and warm-seeded searches (iterations >= 1).

Every named match must be the brute-force nearest neighbour under the contract arithmetic at the transform the last
search used. An exclusion bound that is too large would keep a wrong match in the cache and fail in a later iteration.
"""
import numpy as np
import pytest

from cilantro_b200 import synth

pytestmark = pytest.mark.gpu


def _crowded(rng, n):
    """Tight clumps of 40-200 points in a sparse background: the grid is sized for the mean density."""
    sizes = rng.integers(40, 201, size=n // 120)
    centres = rng.uniform(0.0, 1.0, size=(sizes.size, 3))
    clumps = np.concatenate([c + rng.normal(0.0, 0.002, size=(s, 3)) for c, s in zip(centres, sizes)])
    background = rng.uniform(0.0, 1.0, size=(n - clumps.shape[0], 3)) if n > clumps.shape[0] else np.zeros((0, 3))
    return np.concatenate([clumps, background]).astype(np.float32)


def _slabs(rng, n):
    """Two thin slabs far apart in z: every row between them is empty."""
    p = rng.uniform(0.0, 1.0, size=(n, 3))
    p[:, 2] = np.where(rng.random(n) < 0.5, 0.0, 0.8) + 0.01 * p[:, 2]
    return p.astype(np.float32)


def _lattice(m):
    """Points on a 1/8 lattice (exact in fp32)."""
    g = np.arange(m, dtype=np.float32) / np.float32(8.0)
    return np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)


def _cases():
    rng = np.random.default_rng(17)
    dst = _crowded(rng, 30000)
    src = (dst[rng.permutation(dst.shape[0])[:20000]] + rng.normal(0.0, 0.003, size=(20000, 3))).astype(np.float32)
    yield "crowded", dst, src, 0.05
    dst = _slabs(rng, 30000)
    src = (dst[rng.permutation(dst.shape[0])[:20000]] + rng.normal(0.0, 0.004, size=(20000, 3))).astype(np.float32)
    yield "slabs", dst, src, 0.05
    lat = _lattice(24)
    h = np.float32(1.0 / 16.0)
    # midpoints of edges (2-way ties), face centres (4-way) and cell centres (8-way), plus the lattice points
    offs = np.array([[h, 0, 0], [0, h, 0], [h, h, 0], [0, h, h], [h, h, h], [0, 0, 0]], np.float32)
    src = (lat[rng.permutation(lat.shape[0])[:6000]][:, None, :] + offs[None]).reshape(-1, 3).astype(np.float32)
    yield "lattice", lat, src, 0.15
    dst = rng.uniform(0.0, 1.0, size=(30000, 3)).astype(np.float32)
    src = rng.uniform(-0.3, 1.3, size=(20000, 3)).astype(np.float32)  # a shell of queries outside the grid
    yield "outside", dst, src, 0.05


CASES = {name: (dst, src, max_d) for name, dst, src, max_d in _cases()}


@pytest.mark.parametrize("iters", [1, 2, 5])
@pytest.mark.parametrize("name", sorted(CASES))
def test_loop_cache_matches_brute_force(cb, ctx, orc, name, iters):
    dst, src, max_d = CASES[name]
    icp = cb.Icp(ctx, cb.Cloud(ctx, dst), cb.Cloud(ctx, src))
    max_d2 = np.float32(max_d**2)
    icp.estimate(metric="p2p", max_iter=iters, tol=0.0, max_d2=max_d2, timing=0)
    T_search, near, searched = icp.loop_cache()
    assert (searched == src.shape[0]) if iters == 1 else (searched <= src.shape[0])
    idx, d2 = orc.BruteKnn(dst).query(orc.transform_points(T_search, src), np.float32(3.0e38))
    inside = d2 < max_d2
    assert inside.any()
    assert np.array_equal(near[inside], idx[inside])
    named = (~inside) & (near >= 0)
    assert np.array_equal(near[named], idx[named])


def test_wide_search_matches_on_the_benchmark_pair(cb, ctx, orc):
    """A warm-seeded run on the benchmark's kind of input, every iteration's cache against brute force."""
    dst, src, _, _ = synth.icp_pair(60000, seed=21, noise=0.001, with_normals=False)
    icp = cb.Icp(ctx, cb.Cloud(ctx, dst), cb.Cloud(ctx, src))
    max_d2 = np.float32(0.02**2)
    knn = orc.BruteKnn(dst)
    for iters in (1, 2, 3, 5):
        icp.estimate(metric="p2p", max_iter=iters, tol=0.0, max_d2=max_d2, timing=0)
        T_search, near, _ = icp.loop_cache()
        idx, d2 = knn.query(orc.transform_points(T_search, src), np.float32(3.0e38))
        inside = d2 < max_d2
        assert np.array_equal(near[inside], idx[inside]), iters
