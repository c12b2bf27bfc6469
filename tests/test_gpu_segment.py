"""cb_cloud_segment (ConnectedComponentExtraction3f::segment) on the device: identical to the oracle (cluster CSR,
point -> cluster map, cluster count) for every neighbourhood spec x evaluator kind x {all seeds, seed list}; the
analytic answer of synth.segment_scene; a 1-2 M-point check against scipy on the cb_radius_search graph; a 1 M-point
polyline (one component of diameter 10^6); determinism; the C++ shim and the example program."""
import os

import numpy as np
import pytest

import cxx
import segment_ref as ref

pytestmark = pytest.mark.gpu

ROOT = cxx.ROOT

SPECS = {"radius": (0, 1.0), "knn": (8, 0.0), "knn_in_radius": (8, 1.0)}  # radius2 in units of the spacing^2


@pytest.fixture(scope="module")
def seg(orc):
    from oracle import segment

    return segment


@pytest.fixture(scope="module")
def scene():
    from cilantro_b200 import synth

    s = synth.segment_scene(30000, seed=2)
    rng = np.random.default_rng(9)
    # a colour per object plus small noise; one plate gets two colour halves
    base = rng.random((s["objects"], 3)).astype(np.float32)
    col = base[s["object"]] + 0.01 * rng.standard_normal((s["points"].shape[0], 3)).astype(np.float32)
    half = (s["object"] == 1) & (s["points"][:, 0] > 0.7)
    col[half] += 0.5
    s["colors"] = col.astype(np.float32)
    return s


def evaluators(h):
    """(name, kwargs) for every evaluator kind; thresholds in the scene's spacing."""
    d = float(np.float32((1.2 * h) ** 2))
    out = []
    for terms in range(8):
        for strict, angle in ((False, 0.05), (True, -0.05)) if terms & 2 else ((terms in (3, 6, 7), 0.0),):
            out.append((f"terms{terms}{'s' if strict else ''}",
                        dict(terms=terms, max_distance=d, max_angle=angle, color_thresh=0.1, angle_strict=strict)))
    return out


def run_both(cb, ctx, seg, pts, spec_k, spec_r2, ev, normals=None, colors=None, seeds=None, nbhd=None, cloud=None,
             device_normals=False, min_size=1, max_size=2**64 - 1):
    cloud = cloud or cb.Cloud(ctx, pts, normals if device_normals else None)
    got = cloud.segment(k=spec_k, radius2=spec_r2, normals=None if device_normals else normals, colors=colors, seeds=seeds,
                        min_size=min_size, max_size=max_size, **ev)
    want = seg.connected_components(pts, k=spec_k, radius2=spec_r2, normals=normals, colors=colors, seeds=seeds,
                                    min_size=min_size, max_size=max_size, nbhd=nbhd, **ev)
    return got, want


@pytest.mark.parametrize("spec", sorted(SPECS))
def test_parity_with_the_oracle_on_the_scene(cb, ctx, seg, scene, spec):
    pts, nrm, col, h = scene["points"], scene["normals"], scene["colors"], scene["spacing"]
    k, r = SPECS[spec]
    r2 = float(np.float32((1.5 * h) ** 2 * r)) if r > 0 else 0.0
    nbhd = seg.neighborhoods(pts, k, r2)
    cloud = cb.Cloud(ctx, pts, nrm)
    rng = np.random.default_rng(1)
    seeds = rng.integers(0, pts.shape[0], 40)
    seeds = np.concatenate([seeds, seeds[:5]])[rng.permutation(45)]  # with duplicates
    for name, ev in evaluators(h):
        for sd in (None, seeds):
            for dev in (False, True):
                got, want = run_both(cb, ctx, seg, pts, k, r2, ev, normals=nrm, colors=col, seeds=sd, nbhd=nbhd,
                                     cloud=cloud, device_normals=dev)
                ref.assert_same(got, want, f"{spec} {name} seeds={sd is not None} device_normals={dev}")


def test_known_answer_of_the_scene(cb, ctx, scene):
    pts, nrm, h = scene["points"], scene["normals"], scene["spacing"]
    cloud = cb.Cloud(ctx, pts, nrm)
    r2 = float((1.5 * h) ** 2)
    got = cloud.segment(radius2=r2)
    assert got["num_clusters"] == scene["objects"]
    want = np.sort(np.bincount(scene["object"]))[::-1]
    assert np.array_equal(np.diff(got["offsets"]), want)
    for c in range(got["num_clusters"]):
        assert np.unique(scene["object"][got["points"][got["offsets"][c]:got["offsets"][c + 1]]]).size == 1
    got = cloud.segment(radius2=r2, terms=2, max_angle=float(np.float32(2 * np.pi / 180)))
    assert got["num_clusters"] == scene["faces"]
    assert np.array_equal(np.diff(got["offsets"]), np.sort(np.bincount(scene["face"]))[::-1])
    for c in range(got["num_clusters"]):
        assert np.unique(scene["face"][got["points"][got["offsets"][c]:got["offsets"][c + 1]]]).size == 1


def test_parity_on_a_noisy_sheet_with_device_normals(cb, ctx, seg):
    from cilantro_b200 import synth

    pts, _ = synth.surface_cloud(20000, seed=3, noise=0.002)
    cloud = cb.Cloud(ctx, pts)
    nrm = cloud.estimate_normals(k=10, view_point=[0.5, 0.5, 5.0])["normals"]
    for k, r2 in ((0, 0.012**2), (10, 0.0), (10, 0.012**2)):
        nbhd = seg.neighborhoods(pts, k, r2)
        for ev in (dict(terms=2, max_angle=0.15), dict(terms=2, max_angle=-0.1), dict(terms=3, max_distance=1e-4,
                                                                                       max_angle=0.2, angle_strict=True)):
            for sd in (None, [5, 17, 17, 19999, 3]):
                got = cloud.segment(k=k, radius2=r2, seeds=sd, min_size=3, **ev)  # the normals stored in the cloud
                want = seg.connected_components(pts, k=k, radius2=r2, normals=nrm, seeds=sd, min_size=3, nbhd=nbhd, **ev)
                ref.assert_same(got, want, f"k={k} r2={r2} {ev} seeds={sd}")


def test_degenerate_cases(cb, ctx, seg):
    rng = np.random.default_rng(6)
    base = rng.random((3000, 3)).astype(np.float32)
    pts = np.concatenate([base, base[:500], base[100:300]])  # 2- and 3-fold duplicates
    pts[[7, 1200]] = np.nan
    pts = pts[rng.permutation(pts.shape[0])]
    nrm = rng.standard_normal(pts.shape).astype(np.float32)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    nrm[[11, 2000]] = np.nan
    dup_seed = int(np.flatnonzero((pts == pts[np.flatnonzero(np.isfinite(pts[:, 0]))[0]]).all(1))[-1])
    for k, r2 in ((0, 0.003), (4, 0.0), (4, 0.003)):
        nbhd = seg.neighborhoods(pts, k, r2)
        for ev in (dict(), dict(terms=2, max_angle=1.0), dict(terms=2, max_angle=-0.7)):
            for sd in (None, [dup_seed], [dup_seed, 7, 11, 3], []):
                for mn, mx in ((1, 2**64 - 1), (2, 40), (5, 4)):
                    got, want = run_both(cb, ctx, seg, pts, k, r2, ev, normals=nrm, seeds=sd, nbhd=nbhd, min_size=mn,
                                         max_size=mx)
                    ref.assert_same(got, want, f"k={k} {ev} seeds={sd} min={mn} max={mx}")
    one = np.float32([[1, 2, 3]])
    got = cb.Cloud(ctx, one).segment(radius2=1.0)
    assert got["num_clusters"] == 1 and list(got["points"]) == [0]
    got = cb.Cloud(ctx, np.zeros((0, 3), np.float32)).segment(radius2=1.0)
    assert got["num_clusters"] == 0 and list(got["offsets"]) == [0]


def test_argument_errors(cb, ctx):
    cloud = cb.Cloud(ctx, np.random.default_rng(0).random((100, 3)).astype(np.float32))
    for kw in (dict(radius2=0.01, seeds=[100]), dict(radius2=0.01, terms=2), dict(radius2=0.01, terms=4),
               dict(k=257), dict(k=0, radius2=0.0)):
        with pytest.raises(cb.CbError):
            cloud.segment(**kw)
    shard = cb.Cloud(ctx, np.random.default_rng(0).random((100, 3)).astype(np.float32), index_offset=100)
    with pytest.raises(cb.CbError, match="-5"):
        shard.segment(radius2=0.01)


def test_large_cloud_against_scipy_on_the_radius_search_graph(cb, ctx):
    from cilantro_b200 import synth

    s = synth.segment_scene(1_500_000, seed=4)
    pts, nrm, h = s["points"], s["normals"], s["spacing"]
    nrm = nrm + np.float32(0.01) * np.random.default_rng(1).standard_normal(nrm.shape).astype(np.float32)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    r2 = float(np.float32((1.5 * h) ** 2))
    cloud = cb.Cloud(ctx, pts, nrm)
    off, idx, d2 = cb.radius_search(ctx, cloud, cloud, r2)
    src, dst, dd = ref.edges_from_csr(off, idx, d2)
    for ev in (dict(), dict(terms=2, max_angle=0.04), dict(terms=2, max_angle=-0.04)):
        got = cloud.segment(radius2=r2, min_size=10, **ev)
        want = ref.segment(pts.shape[0], src, dst, ref.accept(src, dst, dd, normals=nrm, **ev), min_size=10)
        ref.assert_same(got, want, str(ev))


def test_one_component_of_diameter_a_million(cb, ctx):
    """A helix whose radius links only consecutive points: the union-find must converge along a 10^6-long path."""
    n = 1_000_000
    t = np.arange(n, dtype=np.float64)
    pts = np.stack([np.cos(t * 0.01), np.sin(t * 0.01), t * 1e-4], 1).astype(np.float32)  # pitch 0.063 >> step 0.01
    p64 = pts.astype(np.float64)
    step2 = np.sum(np.diff(p64, axis=0) ** 2, axis=1)
    skip2 = np.sum((p64[2:] - p64[:-2]) ** 2, axis=1)
    r2 = float(np.float32(1.5 * 1.5 * step2.min()))  # consecutive only: the next-but-one is ~2 steps away
    assert step2.max() < 0.9 * r2 and skip2.min() > 1.5 * r2
    cloud = cb.Cloud(ctx, pts)
    got = cloud.segment(radius2=r2)
    assert got["num_clusters"] == 1 and got["offsets"][-1] == n
    assert np.array_equal(got["points"], np.arange(n))


@pytest.mark.parametrize("outliers", [0, 20])
def test_parity_on_the_far_query_path(cb, ctx, seg, outliers):
    """Sweeps that restart on the far path (grid_sweep's reset): a radius spanning ~19 cells of a fine grid, and kNN
    queries from far outliers, with duplicates and seed lists — the held-back position-0 candidate (seeded radius) and the
    k-best list (kNN) must both be cleared on the restart. tools/segment_counters.py shows these inputs restart."""
    from cilantro_b200 import synth

    pts, nrm = synth.segment_far_scene(seed=7, outliers=outliers)
    cloud = cb.Cloud(ctx, pts, nrm)
    specs = ((8, 0.0), (8, 0.3**2)) if outliers else ((0, 0.3**2),)
    dup = int(np.flatnonzero((pts == pts[0]).all(1))[-1])  # an upper duplicate: its position 0 is a lower index
    far = [int(i) for i in np.flatnonzero(np.abs(pts).max(1) > 3.0)]  # the outliers (and their duplicates)
    for k, r2 in specs:
        r2 = float(np.float32(r2))
        nbhd = seg.neighborhoods(pts, k, r2)
        for ev in (dict(), dict(terms=2, max_angle=0.5), dict(terms=3, max_distance=0.01, max_angle=-0.6, angle_strict=True)):
            for sd in (None, [dup], [dup, 3, 3, pts.shape[0] - 1] + far, list(range(0, pts.shape[0], 97))):
                got, want = run_both(cb, ctx, seg, pts, k, r2, ev, normals=nrm, seeds=sd, nbhd=nbhd, cloud=cloud)
                ref.assert_same(got, want, f"outliers={outliers} k={k} {ev} seeds={sd}")


def test_outputs_are_bit_identical_from_run_to_run(cb, ctx, scene):
    pts, nrm, h = scene["points"], scene["normals"], scene["spacing"]
    cloud = cb.Cloud(ctx, pts, nrm)
    rng = np.random.default_rng(8)
    for kw in (dict(radius2=(1.5 * h) ** 2, terms=2, max_angle=0.05), dict(k=8), dict(k=6, radius2=(1.5 * h) ** 2),
               dict(radius2=(1.5 * h) ** 2, seeds=rng.integers(0, pts.shape[0], 20))):
        a, b = cloud.segment(**kw), cloud.segment(**kw)
        for key in ("offsets", "points", "point_to_cluster"):
            assert np.array_equal(a[key], b[key]), (kw, key)


def test_cpp_shim_runs(cb, tmp_path):
    out = cxx.run(cxx.build(os.path.join(ROOT, "tests", "cpp", "test_segment_shim.cpp"),
                            str(tmp_path / "test_segment_shim")))
    assert "all segmentation shim checks passed" in out


def test_example_program_segments_a_synthetic_scene(cb, tmp_path):
    out = cxx.run(cxx.build(os.path.join(ROOT, "examples", "segment_cloud.cpp"), str(tmp_path / "segment_cloud")),
                  cwd=str(tmp_path))
    assert "components found" in out
