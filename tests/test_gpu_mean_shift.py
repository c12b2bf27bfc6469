"""cb_cloud_mean_shift (MeanShift3f::cluster) on the device: with the unity kernel, bit-identical to the oracle
(shifted seeds, modes, iteration count, labels, CSR) on the reference example's recipe, synth.mean_shift_scene (all
seeds and a seed list, plus its known answer), the far-query path, NaN / Inf points and seeds, r2 == 0, duplicates,
thousands of coincident converged seeds, clustering chains, forced multi-batch runs and a downsampled cloud that
never leaves the device; RBF weights within the stated bound; the error cases."""
import os
import subprocess

import numpy as np
import pytest

from cilantro_b200 import synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = os.path.join(ROOT, "include")
LIBDIR = os.path.join(ROOT, "cilantro_b200")

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


def same(got, want):
    for k in KEYS:
        assert np.array_equal(got[k], want[k]), k
    for k in ("shifted_seeds", "modes"):
        assert got[k].shape == want[k].shape, k
        assert bits(got[k]) == bits(want[k]), k


def both(cb, ctx, ms, pts, *args, cloud=None, **kw):
    cloud = cloud or cb.Cloud(ctx, pts)
    got = cloud.mean_shift(*args, **kw)
    want = ms.mean_shift(pts, *args, **kw)
    return got, want


def example_input(seed=4):
    rng = np.random.default_rng(seed)
    centres = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 1.0]], np.float32)
    return np.concatenate([c + 0.1 * rng.standard_normal((500, 3)) for c in centres]).astype(np.float32)


def test_example_recipe(cb, ctx, ms):
    got, want = both(cb, ctx, ms, example_input(), 0.2, 5000, 0.02)
    same(got, want)
    assert got["iterations"] > 1


def test_scene_known_answer(cb, ctx, ms):
    s = synth.mean_shift_scene(8, 400, sigma=0.5, seed=3)
    pts, sg = s["points"], s["sigma"]
    cloud = cb.Cloud(ctx, pts)
    got, want = both(cb, ctx, ms, pts, 2 * sg, 100, 0.2 * sg, cloud=cloud)
    same(got, want)
    assert got["num_clusters"] == 8
    # one cluster per blob, and every mode near its blob's centre: the blobs are point-symmetric, but a flat-kernel seed
    # stops at a fixed point of its discrete window, within about sigma / sqrt(window size) of the centre (DESIGN §4.11)
    assert len(set(zip(got["point_to_cluster"], s["blob"]))) == 8
    err = np.linalg.norm(got["modes"][got["point_to_cluster"][np.argsort(s["blob"])][::400]] - s["centres"], axis=1)
    assert err.max() < 1e-3 * sg, err.max() / sg
    seeds = pts[::5] + np.float32(0.25 * sg)
    got, want = both(cb, ctx, ms, pts, 2 * sg, 100, 0.2 * sg, seeds=seeds, cloud=cloud)
    same(got, want)
    assert got["num_clusters"] == 8


def test_far_query_path_and_duplicates(cb, ctx, ms):
    pts, _ = synth.segment_far_scene(seed=2, outliers=20)  # 2- and 3-fold duplicates, a fine grid
    rng = np.random.default_rng(5)
    seeds = np.concatenate([pts[::9], rng.uniform(-3.0, 4.0, (40, 3)), [[30.0, -20.0, 5.0]]]).astype(np.float32)
    for radius in (0.3, 0.05):
        got, want = both(cb, ctx, ms, pts, radius, 60, 0.03, seeds=seeds)
        same(got, want)


def test_non_finite_points_seeds_and_zero_radius(cb, ctx, ms):
    pts = example_input(6)[::2].copy()
    pts[5] = [np.nan, 0.0, 0.0]
    pts[9] = [np.inf, 1.0, 0.0]
    pts[11] = [0.0, -np.inf, np.nan]
    seeds = np.concatenate([pts[:40], [[np.nan, 0, 0], [np.inf, 0, 0], [0, -np.inf, 1], [40.0, 0, 0]]]).astype(np.float32)
    cloud = cb.Cloud(ctx, pts)
    got, want = both(cb, ctx, ms, pts, 0.2, 30, 0.02, seeds=seeds, cloud=cloud)
    same(got, want)
    assert got["iterations"] == 30
    got, want = both(cb, ctx, ms, pts, 0.0, 4, 0.02, seeds=seeds, cloud=cloud)
    same(got, want)
    assert np.isnan(got["shifted_seeds"]).all()
    got, want = both(cb, ctx, ms, pts, 0.2, 30, 0.0, seeds=seeds, cloud=cloud)  # cluster_tol 0: singletons
    same(got, want)
    assert got["num_clusters"] == seeds.shape[0]


def test_coincident_converged_seeds(cb, ctx, ms):
    # two dense blobs: thousands of seeds converge onto a handful of bit-identical positions
    s = synth.mean_shift_scene(2, 3000, sigma=1.0, seed=8)
    got, want = both(cb, ctx, ms, s["points"], 2.0, 100, 0.2)
    same(got, want)
    assert got["num_clusters"] == 2
    _, counts = np.unique(got["shifted_seeds"].view(np.uint32).reshape(-1, 3), axis=0, return_counts=True)
    assert counts.max() >= 1000


@pytest.mark.parametrize("reverse", [False, True])
def test_clustering_chain(cb, ctx, ms, reverse):
    tol = 0.1
    n = 1500
    line = np.zeros((n, 3), np.float32)
    line[:, 0] = np.arange(n, dtype=np.float32) * np.float32(0.9 * tol)
    if reverse:
        line = line[::-1].copy()
    got, want = both(cb, ctx, ms, line, 0.5, 0, tol)
    same(got, want)
    assert got["iterations"] == 0 and got["num_clusters"] == (n + 1) // 2


def test_multi_batch_equals_single_batch(cb, ctx, ms, monkeypatch):
    pts = example_input(9)
    cloud = cb.Cloud(ctx, pts)
    one = cloud.mean_shift(0.2, 200, 0.02)
    monkeypatch.setenv("CB_MEAN_SHIFT_PAIR_BUDGET", "1000")
    many = cloud.mean_shift(0.2, 200, 0.02)
    monkeypatch.setenv("CB_MEAN_SHIFT_PAIR_BUDGET", "1")
    single_seed_batches = cloud.mean_shift(0.2, 3, 0.02)
    monkeypatch.delenv("CB_MEAN_SHIFT_PAIR_BUDGET")
    same(many, one)
    same(single_seed_batches, ms.mean_shift(pts, 0.2, 3, 0.02))
    same(one, ms.mean_shift(pts, 0.2, 200, 0.02))


def test_two_runs_identical(cb, ctx):
    s = synth.mean_shift_scene(27, 500, sigma=1.0, seed=4)
    cloud = cb.Cloud(ctx, s["points"])
    a = cloud.mean_shift(2.0, 100, 0.2)
    b = cloud.mean_shift(2.0, 100, 0.2)
    same(a, b)
    assert a["num_clusters"] == 27


def test_downsampled_cloud_stays_on_device(cb, ctx, ms):
    s = synth.mean_shift_scene(4, 2000, sigma=1.0, seed=6)
    ds = cb.Cloud(ctx, s["points"]).grid_downsample(0.25)
    got = ds.mean_shift(2.0, 100, 0.2)
    want = ms.mean_shift(ds.download(), 2.0, 100, 0.2)
    same(got, want)
    assert got["num_clusters"] == 4


@pytest.mark.parametrize("sigma", [1.0, 0.05])
def test_rbf_weights_within_bound(cb, ctx, ms, sigma):
    s = synth.mean_shift_scene(8, 400, sigma=sigma, seed=7)
    got, want = both(cb, ctx, ms, s["points"], 2.0 * sigma, 100, 0.2 * sigma, weight=("rbf", sigma))
    for k in ("offsets", "points", "point_to_cluster", "num_clusters"):
        assert np.array_equal(got[k], want[k]), k
    # expf on the device is not glibc's (<= 2 ulp apart): the weights, and so the seeds, differ in their last bits;
    # later steps start from the perturbed seeds, and seeds still moving when max_iter stops the loop keep what has
    # accumulated (DESIGN §4.11). The bound is relative to the kernel's scale; measured 2.2e-5 sigma at sigma 1 and
    # 2.2e-3 sigma at sigma 0.05.
    for k in ("shifted_seeds", "modes"):
        err = np.abs(got[k].astype(np.float64) - want[k]).max()
        print(f"RBF sigma {sigma} {k}: max |gpu - oracle| = {err / sigma:.3e} sigma, "
              f"iterations {got['iterations']} vs {want['iterations']}")
        assert err < 5e-3 * sigma, (k, err / sigma)


def test_empty_inputs_and_errors(cb, ctx):
    pts = example_input()[:100]
    cloud = cb.Cloud(ctx, pts)
    r = cloud.mean_shift(0.2, 10, 0.02, seeds=np.zeros((0, 3), np.float32))
    assert r["iterations"] == 1 and r["num_clusters"] == 0
    assert cloud.mean_shift(0.2, 0, 0.02, seeds=np.zeros((0, 3), np.float32))["iterations"] == 0
    empty = cb.Cloud(ctx, np.zeros((0, 3), np.float32))
    assert empty.mean_shift(0.2, 10, 0.02)["iterations"] == 1  # no seeds
    with pytest.raises(cb.CbError):
        empty.mean_shift(0.2, 10, 0.02, seeds=pts[:3])
    with pytest.raises(cb.CbError):
        cb.Cloud(ctx, pts, index_offset=100).mean_shift(0.2, 10, 0.02)


def test_large_groups_of_coincident_seeds_are_deduplicated(cb, ctx, ms):
    # 3 x 100 000 bit-identical seeds (and a few loose ones) with max_iter 0: only the first seed of each group of
    # identical coordinates takes part in the clustering sweeps. Without that, every seed of a group would scan the
    # whole group (3 * 10^10 distance tests, tens of seconds); with it the call takes milliseconds.
    pts = example_input()[:200]
    base = np.array([[0.5, 0.5, 0.5], [0.5, 0.5, 0.55], [3.0, 0.0, 0.0]], np.float32)
    rng = np.random.default_rng(3)
    seeds = np.concatenate([np.repeat(base, 100000, axis=0), rng.random((50, 3), dtype=np.float32)])
    seeds = seeds[rng.permutation(seeds.shape[0])]
    cloud = cb.Cloud(ctx, pts)
    cloud.mean_shift(0.2, 0, 0.1, seeds=seeds)  # warm-up
    got = cloud.mean_shift(0.2, 0, 0.1, seeds=seeds)
    want = ms.mean_shift(pts, 0.2, 0, 0.1, seeds=seeds)
    same(got, want)
    sizes = np.diff(got["offsets"])
    assert sizes.max() >= 200000  # the two close groups form one cluster
    print(f"dedup: {seeds.shape[0]} seeds -> {got['num_clusters']} clusters in {got['gpu_ms']:.2f} ms")
    assert got["gpu_ms"] < 1000.0, got["gpu_ms"]


def _cpp_env():
    env = dict(os.environ)
    env.pop("CXX", None)
    env.pop("CC", None)
    return env


def test_cpp_shim_runs(cb, tmp_path):
    exe = str(tmp_path / "test_mean_shift_shim")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", INC, os.path.join(ROOT, "tests", "cpp", "test_mean_shift_shim.cpp"),
                           "-o", exe, "-L", LIBDIR, "-lcilantro_b200", f"-Wl,-rpath,{LIBDIR}"], env=_cpp_env())
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "all mean-shift shim checks passed" in out.stdout


def test_example_program_finds_the_three_blobs(cb, tmp_path):
    exe = str(tmp_path / "mean_shift_cloud")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", INC, os.path.join(ROOT, "examples", "mean_shift_cloud.cpp"),
                           "-o", exe, "-L", LIBDIR, "-lcilantro_b200", f"-Wl,-rpath,{LIBDIR}"], env=_cpp_env())
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300, cwd=str(tmp_path))
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "clusters found" in out.stdout
