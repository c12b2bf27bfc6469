"""cb_cloud_segment at its edges, against the oracle (oracle/segment.py) and the numpy restatement (segment_ref.py):
every kNN instance of segment_kernel (k across the template boundaries, all seeds and a seed list, clouds smaller
than k), ties at the k-th neighbour on integer lattices, directed reachability along a line of growing spacing, every
threshold exactly on its bound, output order and size filters over a million singletons and many equal-size segments,
a 10^5-level BFS, and clouds at the top of the fp32 range. Every input is dyadic, so every boundary is exact."""
import time

import numpy as np
import pytest

import segment_ref as ref
from test_gpu_segment import run_both
from top_range_ref import top_range_cloud

pytestmark = pytest.mark.gpu

F32 = np.float32
K_ALL = (1, 2, 4, 5, 16, 17, 32, 33, 64, 65, 128, 129, 256)


@pytest.fixture(scope="module")
def seg(orc):
    from oracle import segment

    return segment


def lattice_cloud(n, side, seed, dups=0, nan=0):
    """n points on the integer lattice [0, side)^3 (many equal d2), dups exact duplicates, nan NaN points."""
    rng = np.random.default_rng(seed)
    pts = rng.integers(0, side, (n, 3)).astype(F32)
    pts = np.vstack([pts, pts[rng.choice(n, dups)], np.full((nan, 3), np.nan, F32)])
    return pts[rng.permutation(len(pts))]


@pytest.mark.parametrize("r2", [0.0, 4.0], ids=["knn", "knn_in_radius"])
def test_every_kernel_instance_and_ties_at_the_kth_neighbour(cb, ctx, seg, r2):
    t0 = time.perf_counter()
    pts = lattice_cloud(1500, 9, seed=1, dups=60, nan=3)
    small = lattice_cloud(12, 3, seed=2, dups=3)
    cloud, cloud_small = cb.Cloud(ctx, pts), cb.Cloud(ctx, small)
    rng = np.random.default_rng(3)
    seeds = list(rng.integers(0, len(pts), 6)) + [int(np.flatnonzero(np.isnan(pts[:, 0]))[0])]
    assert (seg.neighborhoods(pts, 256, 0.0)[1] == F32(4.0)).any()  # pairs exactly at radius2 = 4
    for k in K_ALL:
        nbhd = seg.neighborhoods(pts, k, r2)
        idx, d2, cnt = nbhd
        if 1 < k and (r2 == 0 or k < cnt.max()):
            # the cut at position k - 1 falls inside a run of equal d2 for many points: the index decides the edge
            full = seg.neighborhoods(pts, min(k + 1, len(pts)), r2)[1]
            assert (full[:, k - 1] == full[:, min(k, full.shape[1] - 1)]).sum() > 100, k
        assert not (d2[np.arange(k)[None, :] < cnt[:, None].astype(np.int64)] >= F32(r2 or np.inf)).any()
        for sd in (None, seeds):
            got, want = run_both(cb, ctx, seg, pts, k, r2, dict(), seeds=sd, nbhd=nbhd, cloud=cloud)
            ref.assert_same(got, want, f"k={k} r2={r2} seeds={sd is not None}")
            if k == 1:  # position 0 is the point or a lower-index twin: no out-edge survives
                assert np.all(np.diff(got["offsets"]) == 1)
            got, want = run_both(cb, ctx, seg, small, k, r2, dict(), seeds=None if sd is None else [0, 5, 5],
                                 cloud=cloud_small)
            ref.assert_same(got, want, f"small k={k} r2={r2} seeds={sd is not None}")
    print(f"[segment-edges] instances r2={r2}: {time.perf_counter() - t0:.3f} s")


def test_directed_reachability_along_a_line(cb, ctx, seg):
    """Spacing i + 1 after point i: with k = 2 every point's one out-edge points to the lower index (point 0's to 1)."""
    n = 300
    x = np.cumsum(np.arange(n, dtype=np.float64))
    pts = np.zeros((n + 2, 3), F32)
    pts[:n, 0] = x
    pts[n:] = np.nan
    gaps = np.diff(pts[:n, 0])
    assert np.all(gaps[1:] > gaps[:-1]) and np.array_equal(pts[:n, 0].astype(np.float64), x)
    cloud = cb.Cloud(ctx, pts)
    nbhd = seg.neighborhoods(pts, 2, 0.0)
    for sd, labelled in (([n - 1], n), ([0], 2), ([n - 1, 0][::-1], n), ([7, 7, 7], 8), ([n, n + 1, 3], 6),
                         ([n + 1], 1), (list(range(n + 1, -1, -37)), None)):
        got, want = run_both(cb, ctx, seg, pts, 2, 0.0, dict(), seeds=sd, nbhd=nbhd, cloud=cloud)
        ref.assert_same(got, want, f"seeds={sd}")
        if labelled is not None:
            assert got["offsets"][-1] == labelled, (sd, got["offsets"][-1])


def _pair_cloud():
    """Point pairs along x at d2 in {1, 2, 4} (exact), normals from the axes (dot 1, 0, -1), colours 0.5 apart."""
    rng = np.random.default_rng(5)
    m = 400
    base = np.column_stack([np.arange(m) * 16.0, np.zeros(m), np.zeros(m)])
    off = np.array([[1.0, 0, 0], [1.0, 1.0, 0], [2.0, 0, 0]])[rng.integers(0, 3, m)]
    pts = np.vstack([base, base + off]).astype(F32)
    axes = np.vstack([np.eye(3), -np.eye(3)])
    nrm = axes[rng.integers(0, 6, 2 * m)].astype(F32)
    col = (rng.integers(0, 3, (2 * m, 3)) * 0.25).astype(F32)
    nrm[rng.choice(2 * m, 10)] = np.nan
    col[rng.choice(2 * m, 10)] = np.nan
    return pts, nrm, col


def test_every_threshold_on_its_bound(cb, ctx, seg):
    pts, nrm, col = _pair_cloud()
    cloud = cb.Cloud(ctx, pts)
    half_pi = F32(np.pi / 2)
    below = lambda v: float(np.nextafter(F32(v), F32(-np.inf)))  # noqa: E731
    above = lambda v: float(np.nextafter(F32(v), F32(np.inf)))  # noqa: E731
    evs = [dict(terms=1, max_distance=d) for d in (1.0, 2.0, above(2.0), 4.0, above(4.0))]
    evs += [dict(terms=2, max_angle=a, angle_strict=s) for a in (0.0, float(half_pi), below(half_pi), above(half_pi),
                                                                   -float(half_pi), -below(half_pi), float(F32(np.pi)))
            for s in (False, True)]
    evs += [dict(terms=4, color_thresh=c) for c in (0.25, above(0.25), 0.5, above(0.5))]
    evs += [dict(terms=7, max_distance=2.0, max_angle=float(half_pi), color_thresh=0.5, angle_strict=s) for s in (0, 1)]
    specs = ((0, 2.0), (0, above(2.0)), (0, 4.0), (4, 2.0), (4, 0.0))
    d2 = seg.neighborhoods(pts, 4, 0.0)[1]
    assert all((d2 == v).any() for v in (1.0, 2.0, 4.0))
    for k, r2 in specs:
        nbhd = seg.neighborhoods(pts, k, r2)
        for ev in evs:
            for sd in (None, [3, 401, 3]):
                got, want = run_both(cb, ctx, seg, pts, k, r2, ev, normals=nrm, colors=col, seeds=sd, nbhd=nbhd,
                                     cloud=cloud)
                ref.assert_same(got, want, f"k={k} r2={r2} {ev} seeds={sd}")


def test_order_of_a_million_singletons(cb, ctx):
    side = 102  # 102^3 > 2^20 lattice points, 1 apart: no pair within radius2 = 0.5
    g = np.arange(side, dtype=F32)
    pts = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    n = pts.shape[0]
    assert n > 2**20
    cloud = cb.Cloud(ctx, pts)
    t0 = time.perf_counter()
    got = cloud.segment(radius2=0.5)
    assert got["num_clusters"] == n and np.array_equal(got["points"], np.arange(n))
    assert np.array_equal(got["point_to_cluster"], np.arange(n))
    perm = np.random.default_rng(6).permutation(n)
    got = cloud.segment(radius2=0.5, seeds=perm)
    assert got["num_clusters"] == n and np.array_equal(got["points"], perm)
    got = cloud.segment(k=4, seeds=perm[: n // 2], min_size=1, max_size=1)
    assert got["num_clusters"] == 0  # kNN: every point reaches its 3 nearest lattice neighbours
    print(f"[segment-edges] {n} singletons: {time.perf_counter() - t0:.3f} s")


def test_equal_sizes_and_exact_size_filters(cb, ctx, seg):
    rng = np.random.default_rng(7)
    sizes = np.concatenate([np.full(300, 2), np.full(200, 3), rng.integers(1, 6, 200)])
    rng.shuffle(sizes)
    pts = np.vstack([np.column_stack([np.full(s, 8.0 * c), np.arange(s), np.zeros(s)]) for c, s in enumerate(sizes)])
    pts = pts[rng.permutation(len(pts))].astype(F32)
    cloud = cb.Cloud(ctx, pts)
    nbhd = seg.neighborhoods(pts, 0, 1.5)
    for mn, mx in ((1, 2**64 - 1), (2, 2), (3, 3), (5, 5), (4, 3), (6, 6)):
        for sd in (None, list(rng.permutation(len(pts))[:500])):
            got, want = run_both(cb, ctx, seg, pts, 0, 1.5, dict(), seeds=sd, nbhd=nbhd, cloud=cloud, min_size=mn,
                                 max_size=mx)
            ref.assert_same(got, want, f"min={mn} max={mx} seeds={sd is not None}")
            if mn == mx and sd is None:
                assert got["num_clusters"] == (sizes == mn).sum()


def test_deep_bfs(cb, ctx):
    """A chain of 10^5 points 1 apart from one seed: the BFS takes one level, one host round trip, per point."""
    n = 100_000
    pts = np.zeros((n, 3), F32)
    pts[:, 0] = np.arange(n)
    cloud = cb.Cloud(ctx, pts)
    cloud.segment(radius2=1.5, seeds=[0, 1])  # builds the index outside the timing
    t0 = time.perf_counter()
    got = cloud.segment(radius2=1.5, seeds=[n - 1])
    dt = time.perf_counter() - t0
    assert got["num_clusters"] == 1 and np.array_equal(got["points"], np.arange(n))
    got = cloud.segment(k=2, seeds=[n // 2])  # equal d2 both ways: every out-edge goes to the lower index
    assert got["num_clusters"] == 1 and np.array_equal(got["points"], np.arange(n // 2 + 1))
    print(f"[segment-edges] {n}-level BFS: {dt:.3f} s")


def test_top_of_the_range(cb, ctx, seg):
    pts = top_range_cloud(seed=8)
    nrm = np.tile(F32([0.0, 0.0, 1.0]), (len(pts), 1))
    cloud = cb.Cloud(ctx, pts)
    for k, r2 in ((0, 0.0625), (0, 1.0), (4, 0.0), (16, 1.0), (256, 0.0)):
        nbhd = seg.neighborhoods(pts, k, r2)
        for ev in (dict(), dict(terms=3, max_distance=0.25, max_angle=0.1)):
            for sd in (None, [0, 5, 5, len(pts) - 1]):
                got, want = run_both(cb, ctx, seg, pts, k, r2, ev, normals=nrm, seeds=sd, nbhd=nbhd, cloud=cloud)
                ref.assert_same(got, want, f"k={k} r2={r2} {ev} seeds={sd}")
                if sd is None and (k, r2) in ((0, 1.0), (4, 0.0)) and not ev:
                    assert got["num_clusters"] < len(pts) // 4  # the columns were linked
