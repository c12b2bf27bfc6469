"""The mean-shift oracle (oracle/mean_shift_oracle.cpp) against an independent numpy / scipy statement
(tests/mean_shift_ref.py): shifted seeds, modes, labels, CSR and iteration count bit for bit, on the reference
example's recipe, explicit seeds, max_iter 0, zero seeds, cluster_tol 0, and NaN / Inf / far seeds."""
import numpy as np
import pytest

import mean_shift_ref as ref
from cilantro_b200 import synth

KEYS = ("offsets", "points", "point_to_cluster", "num_clusters", "iterations")


@pytest.fixture(scope="module")
def ms():
    from oracle import mean_shift

    mean_shift.build()
    return mean_shift


def bits(a):
    """Bit patterns with every NaN as one value: the sign and payload of a NaN that arithmetic creates are the
    hardware's (x86 gives 0xffc00000, the GPU 0x7fffffff); which values are NaN is part of the contract."""
    return np.where(np.isnan(a), np.uint32(0x7fc00000), a.view(np.uint32)).tolist()


def same(a, b):
    for k in KEYS:
        assert np.array_equal(a[k], b[k]), k
    for k in ("shifted_seeds", "modes"):
        assert a[k].shape == b[k].shape, k
        assert bits(a[k]) == bits(b[k]), k


def example_input(seed=4):
    """Three 500-point clusters with spread 0.1 around three centres, like examples/mean_shift.cpp (own RNG)."""
    rng = np.random.default_rng(seed)
    centres = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 1.0]], np.float32)
    return np.concatenate([c + 0.1 * rng.standard_normal((500, 3)) for c in centres]).astype(np.float32)


def test_example_recipe(ms):
    pts = example_input()
    got = ms.mean_shift(pts, 0.2, 5000, 0.02)
    same(got, ref.mean_shift(pts, 0.2, 5000, 0.02))
    assert got["num_clusters"] >= 3 and got["iterations"] > 1


def test_scene_and_explicit_seeds(ms):
    s = synth.mean_shift_scene(3, 400, sigma=0.5, seed=1)
    pts, sg = s["points"], s["sigma"]
    got = ms.mean_shift(pts, 2 * sg, 100, 0.2 * sg)
    same(got, ref.mean_shift(pts, 2 * sg, 100, 0.2 * sg))
    assert got["num_clusters"] == 3
    seeds = pts[::7] + np.float32(0.3 * sg)
    same(ms.mean_shift(pts, 2 * sg, 100, 0.2 * sg, seeds=seeds), ref.mean_shift(pts, 2 * sg, 100, 0.2 * sg, seeds=seeds))


def test_rbf_weights(ms):
    s = synth.mean_shift_scene(3, 100, sigma=1.0, seed=2)
    pts = s["points"]
    got = ms.mean_shift(pts, 2.0, 50, 0.2, weight=("rbf", 1.0))
    want = ref.mean_shift(pts, 2.0, 50, 0.2, rbf_sigma=1.0)
    for k in KEYS:
        assert np.array_equal(got[k], want[k]), k
    # glibc expf in both; numpy's float32 exp may differ in the last bit
    assert np.abs(got["shifted_seeds"] - want["shifted_seeds"]).max() < 1e-4


@pytest.mark.parametrize("max_iter", [0, 1, 3])
def test_few_iterations(ms, max_iter):
    pts = example_input(7)[::3]
    same(ms.mean_shift(pts, 0.2, max_iter, 0.05), ref.mean_shift(pts, 0.2, max_iter, 0.05))


def test_zero_seeds_counts_one_iteration(ms):
    pts = example_input()[:50]
    got = ms.mean_shift(pts, 0.2, 10, 0.02, seeds=np.zeros((0, 3), np.float32))
    assert got["iterations"] == 1 and got["num_clusters"] == 0 and list(got["offsets"]) == [0]
    assert ms.mean_shift(pts, 0.2, 0, 0.02, seeds=np.zeros((0, 3), np.float32))["iterations"] == 0


def test_cluster_tol_zero_gives_singletons(ms):
    pts = example_input()[::5]
    got = ms.mean_shift(pts, 0.2, 100, 0.0)
    same(got, ref.mean_shift(pts, 0.2, 100, 0.0))
    assert got["num_clusters"] == pts.shape[0]


def test_non_finite_and_far_seeds(ms):
    pts = example_input()[::4]
    seeds = np.concatenate([pts[:20], [[np.nan, 0, 0], [np.inf, 0, 0], [0, -np.inf, 1], [50.0, 50.0, 50.0]], pts[20:30]])
    got = ms.mean_shift(pts, 0.2, 40, 0.02, seeds=seeds.astype(np.float32))
    same(got, ref.mean_shift(pts, 0.2, 40, 0.02, seeds=seeds))
    assert got["iterations"] == 40  # a seed that never converges forces max_iter
    bad = got["shifted_seeds"][20:24]
    assert not np.isfinite(bad).all(axis=1).any()
    assert len(set(got["point_to_cluster"][20:24])) == 4  # singletons
    # r2 == 0: every seed lands on NaN
    got0 = ms.mean_shift(pts, 0.0, 5, 0.02)
    same(got0, ref.mean_shift(pts, 0.0, 5, 0.02))
    assert np.isnan(got0["shifted_seeds"]).all() and got0["num_clusters"] == pts.shape[0]


def test_nan_points_are_inert(ms):
    pts = example_input()[::4].copy()
    pts[3] = [np.nan, 0, 0]
    pts[10] = [np.inf, np.inf, 0]
    seeds = pts[np.isfinite(pts).all(axis=1)][:60]
    same(ms.mean_shift(pts, 0.2, 30, 0.02, seeds=seeds), ref.mean_shift(pts, 0.2, 30, 0.02, seeds=seeds))
