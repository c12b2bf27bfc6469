"""The connected-component oracle (oracle/cce_oracle.cpp, a serial restatement of extractConnectedComponents) against an
independent statement of the pinned semantics (tests/segment_ref.py: scipy weakly connected components on the directed
edge graph, numpy BFS reachability for seed lists). CPU only."""
import numpy as np
import pytest

import segment_ref as ref


@pytest.fixture(scope="module")
def seg(orc):
    from oracle import segment

    return segment


def both(seg, pts, seeds=None, min_size=1, max_size=2**64 - 1, k=0, radius2=0.0, **ev):
    """Oracle result and the independent one, on the same brute-force neighbourhoods."""
    pts = np.ascontiguousarray(pts, np.float32)
    idx, d2, cnt = seg.neighborhoods(pts, k, radius2)
    got = seg.connected_components(pts, nbhd=(idx, d2, cnt), seeds=seeds, min_size=min_size, max_size=max_size, **ev)
    src, dst, dd = ref.edges_from_rows(idx, d2, cnt)
    ok = ref.accept(src, dst, dd, **ev)
    want = ref.segment(pts.shape[0], src, dst, ok, seeds=seeds, min_size=min_size, max_size=max_size)
    ref.assert_same(got, want)
    return got


def line(n):
    return np.stack([np.arange(n), np.zeros(n), np.zeros(n)], 1).astype(np.float32)


def test_two_separated_blobs(seg):
    rng = np.random.default_rng(0)
    a = rng.random((60, 3)) * 0.1
    b = rng.random((40, 3)) * 0.1 + 5.0
    pts = np.concatenate([b[:20], a, b[20:]])
    got = both(seg, pts, radius2=0.2**2)
    assert got["num_clusters"] == 2 and list(np.diff(got["offsets"])) == [60, 40]
    assert np.array_equal(got["points"][:60], np.arange(20, 80))


def test_chain_cut_by_a_flipped_normal_and_rejoined_unoriented(seg):
    pts = line(10)
    nrm = np.tile(np.float32([0, 0, 1]), (10, 1))
    nrm[5] = -nrm[5]
    got = both(seg, pts, radius2=1.5**2, terms=2, max_angle=0.1, normals=nrm)
    assert list(np.diff(got["offsets"])) == [5, 4, 1] and list(got["points"]) == [0, 1, 2, 3, 4, 6, 7, 8, 9, 5]
    got = both(seg, pts, radius2=1.5**2, terms=2, max_angle=-0.1, normals=nrm)
    assert got["num_clusters"] == 1 and got["offsets"][-1] == 10
    # the combined evaluator's strict comparison: angle 0 < 0 fails, so nothing is joined
    got = both(seg, pts, radius2=1.5**2, terms=3, max_distance=10.0, max_angle=0.0, angle_strict=True, normals=nrm)
    assert got["num_clusters"] == 10


@pytest.mark.parametrize("k,radius2", [(1, 0.0), (2, 0.0), (3, 0.0), (5, 0.05), (4, 0.0)])
def test_asymmetric_knn_neighbourhoods(seg, k, radius2):
    rng = np.random.default_rng(k)
    pts = rng.random((400, 3)).astype(np.float32)
    both(seg, pts, k=k, radius2=radius2)
    both(seg, pts, k=k, radius2=radius2, seeds=rng.integers(0, 400, 7))


def test_duplicates_and_the_skipped_position_zero(seg):
    # 0 and 1 coincide; N(1) = [0, 1]: position 0 is the lower-index duplicate, so 1 -> 0 is not an edge
    pts = np.float32([[0, 0, 0], [0, 0, 0], [5, 5, 5], [5, 5, 5], [5, 5, 5], [9, 9, 9]])
    got = both(seg, pts, radius2=0.5, seeds=[1])
    assert got["num_clusters"] == 1 and list(got["points"]) == [1] and got["point_to_cluster"][0] == 1
    got = both(seg, pts, radius2=0.5, seeds=[0])
    assert list(got["points"]) == [0, 1]
    got = both(seg, pts, radius2=0.5, seeds=[4, 3])
    assert list(got["points"]) == [3, 4]  # 4 reaches 4 only (its position 0 is 2); 3 reaches 4
    got = both(seg, pts, radius2=0.5)
    assert list(np.diff(got["offsets"])) == [3, 2, 1]
    both(seg, pts, k=2)
    both(seg, pts, k=2, seeds=[4, 4, 1, 5])
    rng = np.random.default_rng(3)
    base = rng.random((100, 3)).astype(np.float32)
    pts = np.concatenate([base, base[:30], base[10:20]])[rng.permutation(140)]
    for seeds in (None, rng.integers(0, 140, 10)):
        both(seg, pts, radius2=0.01, seeds=seeds)
        both(seg, pts, k=3, seeds=seeds)


def test_nan_points_and_nan_normals(seg):
    rng = np.random.default_rng(4)
    pts = rng.random((200, 3)).astype(np.float32)
    pts[[3, 50]] = np.nan
    nrm = rng.standard_normal((200, 3)).astype(np.float32)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    nrm[[7, 90]] = np.nan
    got = both(seg, pts, radius2=0.03)
    for p in (3, 50):
        c = got["point_to_cluster"][p]
        assert np.diff(got["offsets"])[c] == 1  # a NaN point is a singleton
    both(seg, pts, radius2=0.03, terms=2, max_angle=1.0, normals=nrm)
    both(seg, pts, radius2=0.03, terms=2, max_angle=-0.5, normals=nrm, seeds=[3, 7, 11])
    both(seg, pts, k=5, terms=2, max_angle=1.2, normals=nrm)


def test_min_max_filters(seg):
    pts = np.concatenate([line(7), line(3) + 100, line(5) + 200, line(1) + 300])
    got = both(seg, pts, radius2=1.5**2)
    assert list(np.diff(got["offsets"])) == [7, 5, 3, 1]
    got = both(seg, pts, radius2=1.5**2, min_size=3, max_size=5)
    assert list(np.diff(got["offsets"])) == [5, 3] and (got["point_to_cluster"][:7] == 2).all()
    got = both(seg, pts, radius2=1.5**2, max_size=6)
    assert list(np.diff(got["offsets"])) == [5, 3, 1]
    both(seg, pts, radius2=1.5**2, min_size=8)


def test_equal_size_ties(seg):
    pts = np.concatenate([line(4) + 300, line(4), line(4) + 100, line(4) + 200])
    got = both(seg, pts, radius2=1.5**2)
    assert list(got["points"][::4]) == [0, 4, 8, 12]
    # seed order decides: the segment holding the earliest seed-list entry comes first
    got = both(seg, pts, radius2=1.5**2, seeds=[9, 13, 2, 5, 10])
    assert list(got["points"][::4]) == [8, 12, 0, 4]


def test_evaluator_kinds(seg):
    rng = np.random.default_rng(5)
    pts = rng.random((500, 3)).astype(np.float32)
    nrm = rng.standard_normal((500, 3)).astype(np.float32)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    col = rng.random((500, 3)).astype(np.float32)
    for terms in range(8):
        for strict in (False, True):
            ev = dict(terms=terms, max_distance=0.004, max_angle=0.9, color_thresh=0.5, angle_strict=strict, normals=nrm,
                      colors=col)
            both(seg, pts, radius2=0.01, **ev)
            both(seg, pts, k=6, seeds=[0, 499, 7, 7], **ev)


def test_degenerate_inputs(seg):
    empty = np.zeros((0, 3), np.float32)
    got = seg.connected_components(empty, radius2=1.0)
    assert got["num_clusters"] == 0 and list(got["offsets"]) == [0]
    got = both(seg, np.float32([[1, 2, 3]]), radius2=1.0)
    assert got["num_clusters"] == 1 and list(got["points"]) == [0]
    got = both(seg, line(5), radius2=2.0, seeds=[])
    assert got["num_clusters"] == 0 and (got["point_to_cluster"] == 0).all()
