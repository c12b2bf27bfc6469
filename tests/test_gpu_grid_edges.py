"""Grid searches against brute force where the uniform grid goes wrong: extreme coordinate scales and offsets, cell edges
whose square leaves the fp32 range, axis-capped grids, cells of thousands to hundreds of thousands of points, queries
on cell faces and reference points exactly on the search bound.

Every grid consumer is compared with orc.BruteKnn (the fp32 arithmetic contract, lowest index wins exact ties):
cb_knn1_radius, cb_find_correspondences, cb_knn_radius (at the template boundaries of knn_k.cu), cb_radius_search
and k-mode normals. Indices and counts must be identical, squared distances and covariances bit-identical. Each case
first checks through Cloud.grid_info() that it built the grid it is about (DESIGN §4.1), and prints its wall time.
"""
import time

import numpy as np
import pytest

from cilantro_b200 import synth
from conftest import frob

pytestmark = pytest.mark.gpu

F32 = np.float32
FMAX = float(np.finfo(np.float32).max)
FMIN = float(np.finfo(np.float32).tiny)
HS2_OVERFLOW_EDGE = 1.8446744e19  # cell edge whose square (times (1 - 2^-10)^2) exceeds FLT_MAX
K_BOUNDARIES = (1, 4, 5, 16, 17, 32, 33, 64, 65, 128, 129, 256)
HUGE_CELL = 1 << 16


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _report(name, t0):
    print(f"[grid-edges] {name}: {time.perf_counter() - t0:.3f} s")


def _approx_cell_counts(pts, info):
    """Points per cell of the grid grid_info() describes (float64 restatement of the binning: exact away from faces,
    which is all the occupancy assertions need)."""
    h = float(info["cell_edge"])
    fin = np.isfinite(pts).all(axis=1)
    p = pts[fin].astype(np.float64)
    org = p.min(axis=0) - h
    dims = np.array(info["dims"])
    c = np.clip(np.floor((p - org) / h).astype(np.int64), 0, dims - 1)
    _, cnt = np.unique((c[:, 2] * dims[1] + c[:, 1]) * dims[0] + c[:, 0], return_counts=True)
    return cnt


def _check(cb, ctx, orc, ref_pts, qry_pts, T=None, max_d2=FMAX, ks=(1, 16), r2=None, corr_d2=None, ref=None):
    """Every search flavour against brute force; returns the device results for further comparison."""
    ref = ref if ref is not None else cb.Cloud(ctx, ref_pts)
    q = cb.Cloud(ctx, qry_pts)
    qt = orc.transform_points(T, qry_pts) if T is not None else qry_pts
    brute = orc.BruteKnn(ref_pts)
    out = {}
    idx, d2 = cb.knn1_radius(ctx, ref, q, T, max_d2)
    oi, od = brute.query(qt, max_d2)
    assert np.array_equal(idx, oi), f"knn1: {(idx != oi).sum()} of {idx.size} index mismatches"
    assert np.array_equal(_bits(d2), _bits(od)), f"knn1: {(_bits(d2) != _bits(od)).sum()} d2 differ bitwise"
    out["knn1"] = (idx, d2)
    if corr_d2 is not None:
        i1, i2, v = cb.find_correspondences(ctx, ref, q, T, corr_d2)
        o1, o2, ov = orc.find_correspondences(T if T is not None else orc.identity(), qry_pts, brute, corr_d2)
        assert np.array_equal(i1, o1) and np.array_equal(i2, o2), f"correspondences: {i1.size} vs {o1.size} pairs"
        assert np.array_equal(_bits(v), _bits(ov))
        out["corr"] = (i1, i2, v)
    for k in ks:
        kidx, kd2, cnt = cb.knn_radius(ctx, ref, q, k, T, max_d2)
        bi, bd, bc = brute.neighborhoods(qt, k, max_d2)
        assert np.array_equal(cnt, bc), f"k={k}: {(cnt != bc).sum()} count mismatches"
        assert np.array_equal(kidx, bi), f"k={k}: {(kidx != bi).any(axis=1).sum()} rows with index mismatches"
        used = np.arange(k)[None, :] < cnt[:, None]
        assert np.array_equal(_bits(kd2[used]), _bits(bd[used])), f"k={k}: d2 differ bitwise"
        out[k] = (kidx, kd2, cnt)
    if r2 is not None:
        off, ridx, rd2 = cb.radius_search(ctx, ref, q, r2, T=T)
        _, _, bc = brute.neighborhoods(qt, 0, r2, stride=1)
        bi, bd, bc = brute.neighborhoods(qt, 0, r2, stride=max(1, int(bc.max()) if bc.size else 1))
        assert np.array_equal(np.diff(off), bc.astype(np.int64)), f"radius: {(np.diff(off) != bc).sum()} count mismatches"
        used = np.arange(bi.shape[1])[None, :] < bc[:, None].astype(np.int64)
        assert np.array_equal(ridx, bi[used]) and np.array_equal(_bits(rd2), _bits(bd[used]))
        out["radius"] = (off, ridx, rd2)
    return out


def _check_normals_k(cb, ctx, orc, pts, k):
    got = cb.Cloud(ctx, pts).estimate_normals(k=k, view_point=[0.5, 0.5, 10.0], want_cov=True)
    want = orc.estimate_normals(pts, orc.BruteKnn(pts), k=k, view_point=[0.5, 0.5, 10.0])
    assert np.array_equal(_bits(got["cov6"]), _bits(want[2])), f"normals k={k}: covariances differ bitwise"
    return got


# ---- power-of-two scale sweep ----------------------------------------------------------------------------------------
def _clustered_scene(seed):
    rng = np.random.default_rng(seed)
    centres = rng.random((3, 3))
    ref = np.vstack([c + 0.02 * rng.standard_normal((4000, 3)) for c in centres] + [rng.random((8000, 3))])
    qry = np.vstack([ref[rng.choice(len(ref), 2000)] + 0.005 * rng.standard_normal((2000, 3)),
                     rng.random((1500, 3)) * 1.4 - 0.2, rng.random((500, 3)) * 11 - 5])
    return ref.astype(F32), qry.astype(F32)


def test_power_of_two_scale_sweep(cb, ctx, orc):
    """Scaling a cloud, its queries and T's translation by 2^e is exact in fp32: inside the normal range the grid,
    the indices and the d2 (times 4^e) are those of e = 0. Below it (subnormal d2) and beyond it (a cell edge past
    1.84e19, where h_safe^2 overflows fp32) the results must still equal brute force."""
    ref0, qry0 = _clustered_scene(1)
    T0 = synth.rigid_from_axis_angle([1, 2, 3], 0.3, [0.05, -0.03, 0.02]).astype(F32)
    sub = slice(0, 4000, 8)  # 500 queries for the k sweep and the radius lists
    base = None
    e_h = None
    for e in (0, -60, -40, -20, 20, 40, 60, "h"):
        if e == "h":  # the first e whose cell edge passes the fp32 overflow of h_safe^2
            e = e_h = int(np.ceil(np.log2(HS2_OVERFLOW_EDGE * 1.01 / base["edge"])))
        t0 = time.perf_counter()
        s = 2.0 ** e
        ref, qry = (ref0 * s).astype(F32), (qry0 * s).astype(F32)
        T = T0.copy()
        T[:, 3] = (T0[:, 3].astype(np.float64) * s).astype(F32)
        assert np.array_equal(ref.astype(np.float64), ref0.astype(np.float64) * s)  # the scaling is exact
        cl = cb.Cloud(ctx, ref)
        info = cl.grid_info()
        if base is not None:
            assert info["dims"] == base["dims"] and info["cell_edge"] == F32(base["edge"] * s), (e, info)
        bound = F32(min(0.03**2 * 4.0**e, FMAX))  # exactly 4^e times the e = 0 bound in the normal range
        out = _check(cb, ctx, orc, ref, qry, T=T, max_d2=FMAX, ks=(), ref=cl)
        bnd = _check(cb, ctx, orc, ref, qry, T=T, max_d2=bound, ks=(), corr_d2=bound, ref=cl)
        ks = _check(cb, ctx, orc, ref, qry[sub], T=T, max_d2=FMAX, ks=K_BOUNDARIES, ref=cl,
                    r2=F32(min(0.02**2 * 4.0**e, FMAX)))
        if e in (-40, 0, 40):
            _check_normals_k(cb, ctx, orc, ref, 16)
        if e == 0:
            base = dict(edge=info["cell_edge"], dims=info["dims"], out=out, bnd=bnd, ks=ks)
        elif -40 <= e <= 60:
            # normal range: the very same answers, d2 scaled exactly
            def same(a, b):
                ia, da = a
                ib, db = b
                assert np.array_equal(ia, ib), (e, (ia != ib).sum())
                want = (db.astype(np.float64) * 4.0**e).astype(F32)
                assert np.array_equal(_bits(da), _bits(want)), e

            same(out["knn1"], base["out"]["knn1"])
            same(bnd["knn1"], base["bnd"]["knn1"])
            assert np.array_equal(bnd["corr"][1], base["bnd"]["corr"][1])
            for k in K_BOUNDARIES:
                assert np.array_equal(ks[k][2], base["ks"][k][2]), (e, k)
                same(ks[k][:2], base["ks"][k][:2])
        elif e == -60:
            assert (out["knn1"][1] < FMIN).any()  # the subnormal regime was reached
        else:
            assert (info["cell_edge"] * (1 - 2**-10)) ** 2 > FMAX  # the regime the hs2 clamp is about
        _report(f"scale 2^{e} (cell edge {info['cell_edge']:.3e}, dims {info['dims']})", t0)
    assert e_h is not None and e_h > 60


# ---- cell edges past the overflow of h_safe^2 ------------------------------------------------------------------------
def test_cell_edge_beyond_fp32_square_two_clusters(cb, ctx, orc):
    """Two 2000-point clusters spanning 1e20 at the two ends of a 4e22 rod: the occupancy loop ends at the axis cap
    with a cell edge of ~4.9e19, whose square is not a finite fp32. Neighbour spacing ~8e18 keeps the nearest d2
    finite (~6e37), and each cluster spans about two cells per axis, so many nearest neighbours lie across a face."""
    t0 = time.perf_counter()
    rng = np.random.default_rng(7)
    span, length = 1e20, 4e22
    far = np.array([length - span, 0.0, 0.0])
    ref = np.vstack([rng.random((2000, 3)) * span, far + rng.random((2000, 3)) * span]).astype(F32)
    cl = cb.Cloud(ctx, ref)
    info = cl.grid_info()
    h = info["cell_edge"]
    assert HS2_OVERFLOW_EDGE < h < 1e20 and max(info["dims"]) > 512, info
    # queries inside both cluster boxes, and on / next to every cell face crossing them
    qa = rng.random((1000, 3)) * span
    qb = far + rng.random((1000, 3)) * span
    org = ref.astype(np.float64).min(axis=0) - h
    faces = []
    for lo3 in (np.zeros(3), far):
        for ax in range(3):
            lo = lo3[ax]
            k0, k1 = int(np.ceil((lo - org[ax]) / h)), int(np.floor((lo + span - org[ax]) / h))
            for k in range(k0, k1 + 1):
                f = F32(org[ax] + k * h)
                for v in (f, np.nextafter(f, F32(np.inf)), np.nextafter(f, F32(-np.inf))):
                    q = lo3 + rng.random((20, 3)) * span
                    q[:, ax] = v
                    faces.append(q)
    qry = np.vstack([qa, qb] + faces).astype(F32)
    print(f"[grid-edges] two clusters: grid_info {info}, {len(faces) * 20} face queries")
    _check(cb, ctx, orc, ref, qry, max_d2=FMAX, ks=(1, 4, 16), r2=F32(1e38), corr_d2=F32(1e38), ref=cl)
    _check_normals_k(cb, ctx, orc, ref, 16)
    _report("two clusters, cell edge past sqrt(FLT_MAX)", t0)


# ---- large offsets ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("offset", [1e3, 1e5, 1e7])
def test_large_offsets(cb, ctx, orc, offset):
    """A 0.1-10-unit scene moved 1e3 / 1e5 / 1e7 from the origin: fp32 quantises the coordinates (to 1 unit at 1e7,
    where points collapse into exact duplicates and ties). With and without a rigid T about the scene centre."""
    t0 = time.perf_counter()
    rng = np.random.default_rng(int(np.log10(offset)))
    scene = np.vstack([rng.random((10000, 3)) * 10] + [c + 0.1 * rng.standard_normal((1000, 3))
                                                        for c in rng.random((5, 3)) * 10])
    ref = (scene + offset).astype(F32)
    qry = (scene[rng.choice(len(scene), 3000)] + 0.05 * rng.standard_normal((3000, 3)) + offset).astype(F32)
    cl = cb.Cloud(ctx, ref)
    info = cl.grid_info()
    assert min(info["dims"]) >= 10, info
    ulp = float(np.spacing(F32(offset + 10)))
    r = max(0.2, 1.5 * ulp)
    r2 = F32(r * r)
    R = synth.rigid_from_axis_angle([0.3, -1, 0.5], 0.2, [0, 0, 0])[:, :3]
    c = np.full(3, offset + 5.0)
    T = np.hstack([R, (c - R @ c)[:, None]]).astype(F32)
    for TT in (None, T):
        _check(cb, ctx, orc, ref, qry, T=TT, max_d2=FMAX, ks=(1, 16, 33), ref=cl)
        _check(cb, ctx, orc, ref, qry, T=TT, max_d2=r2, ks=(16,), r2=r2, corr_d2=r2, ref=cl)
    _check_normals_k(cb, ctx, orc, ref, 16)
    _report(f"offset {offset:g} (fp32 spacing {ulp:g}, grid {info})", t0)


# ---- anisotropy and the axis cap -------------------------------------------------------------------------------------
def _anisotropic(case, rng):
    if case == "rod":
        return (rng.random((30000, 3)) * [1e4, 1, 1]).astype(F32)
    if case == "sheet":
        return (rng.random((30000, 3)) * [1, 1, 1e-6]).astype(F32)
    pts, _ = synth.surface_cloud(30000, seed=5)
    return np.vstack([pts, [[1e4, 0.5, 0.5]]]).astype(F32)  # a scan and one outlier 1e4 extents away


@pytest.mark.parametrize("case", ["rod", "sheet", "outlier"])
def test_anisotropic_and_axis_capped_grids(cb, ctx, orc, case):
    """A 1e4 x 1 x 1 rod and a scan with a far outlier hit the 1024-cells-per-axis cap (the 1.26 growth loop of
    ensure_index then leaves the long axis between 1024 / 1.26 and 1024 cells); a 1 x 1 x 1e-6 sheet is one cell
    thick. The scan behind the outlier collapses into a few cells of thousands of points."""
    t0 = time.perf_counter()
    rng = np.random.default_rng(3)
    ref = _anisotropic(case, rng)
    cl = cb.Cloud(ctx, ref)
    info = cl.grid_info()
    dims = info["dims"]
    if case == "sheet":
        assert dims[2] == 3 and min(dims[:2]) > 50, info
    else:
        assert 1024 / 1.26 <= max(dims) <= 1024, info  # capped
        if case == "rod":
            assert dims[1] == dims[2] == 3, info
        else:
            assert _approx_cell_counts(ref, info).max() > 3000, info
    ext = ref.max(axis=0).astype(np.float64) - ref.min(axis=0)
    qry = np.vstack([ref[rng.choice(len(ref), 3000)] + 1e-3 * rng.standard_normal((3000, 3)) * np.clip(ext, 1e-3, 1),
                     ref.min(axis=0) + rng.random((1000, 3)) * ext]).astype(F32)
    r2 = F32(0.05**2)
    _check(cb, ctx, orc, ref, qry, max_d2=FMAX, ks=(1, 16, 17), ref=cl)
    _check(cb, ctx, orc, ref, qry, max_d2=r2, ks=(16,), r2=r2, corr_d2=r2, ref=cl)
    _check_normals_k(cb, ctx, orc, ref, 8)
    _report(f"{case} (grid {info})", t0)


# ---- cell occupancy ----------------------------------------------------------------------------------------------------
def test_big_cells_in_a_sparse_cloud(cb, ctx, orc):
    """A dense 10 k-point cluster inside a sparse cloud: the sparse points keep the cell edge coarse, so the cluster
    fills cells of thousands of points (the block-per-cell rank sort of the grid build)."""
    t0 = time.perf_counter()
    rng = np.random.default_rng(11)
    ref = np.vstack([rng.random((20000, 3)) * 10, 5.3 + 0.0005 * rng.standard_normal((10000, 3))]).astype(F32)
    ref = ref[rng.permutation(len(ref))]
    cl = cb.Cloud(ctx, ref)
    info = cl.grid_info()
    big = _approx_cell_counts(ref, info).max()
    assert 1000 < big <= HUGE_CELL, (big, info)
    qry = np.vstack([5.3 + 0.001 * rng.standard_normal((2000, 3)), rng.random((2000, 3)) * 10]).astype(F32)
    _check(cb, ctx, orc, ref, qry, max_d2=FMAX, ks=(1, 16, 33, 65), ref=cl)
    r2 = F32(0.0004**2)
    _check(cb, ctx, orc, ref, qry, max_d2=r2, ks=(), r2=r2, corr_d2=r2, ref=cl)
    _check_normals_k(cb, ctx, orc, ref, 16)
    _report(f"big cells (largest ~{big} points, grid {info})", t0)


def test_huge_cell_collapsed_by_an_outlier(cb, ctx, orc):
    """200 k points in the unit cube and one point 1e5 away: the axis cap makes the cell edge ~120, so the whole
    cube is one cell of 200 k points (beyond the 65 536 of the rank sort). Exact against brute force; the device
    time of the collapsed search (O(queries x cell size) by design) is printed."""
    rng = np.random.default_rng(12)
    ref = np.vstack([rng.random((200000, 3)), [[1e5, 1e5, 1e5]]]).astype(F32)
    cl = cb.Cloud(ctx, ref)
    info = cl.grid_info()
    big = _approx_cell_counts(ref, info).max()
    assert big > 150000, (big, info)
    t0 = time.perf_counter()
    qry = np.vstack([ref[rng.choice(200000, 1500)] + 1e-4 * rng.standard_normal((1500, 3)),
                     rng.random((500, 3)) * 1.2 - 0.1]).astype(F32)
    _check(cb, ctx, orc, ref, qry, max_d2=FMAX, ks=(1, 17), ref=cl)
    r2 = F32(0.01**2)
    _check(cb, ctx, orc, ref, qry, max_d2=r2, ks=(), r2=r2, corr_d2=r2, ref=cl)
    _report(f"huge cell exactness (largest ~{big} points, grid {info})", t0)
    many = cb.Cloud(ctx, rng.random((20000, 3)).astype(F32))
    idx, _ = cb.knn1_radius(ctx, cl, many, None, FMAX)
    t0 = time.perf_counter()
    idx2, _ = cb.knn1_radius(ctx, cl, many, None, FMAX)
    print(f"[grid-edges] collapsed grid: 1-NN of 20000 queries in a {big}-point cell: "
          f"{(time.perf_counter() - t0) * 1e3:.1f} ms")
    assert np.array_equal(idx, idx2)


def test_huge_cells_give_bit_identical_reruns(cb, ctx, orc):
    """Sums taken in cell order over a cloud with a cell of more than 65 536 points: radius-mode normals and a
    10-iteration ICP (both loops) repeat bit for bit on freshly built clouds, and the ICP agrees with the oracle."""
    t0 = time.perf_counter()
    rng = np.random.default_rng(13)
    pts, _ = synth.surface_cloud(70000, seed=13)
    cloud = np.vstack([pts, [[1e4, 1e4, 1e4]]]).astype(F32)
    runs = []
    for _ in range(2):
        c = cb.Cloud(ctx, cloud)
        info = c.grid_info()
        runs.append(c.estimate_normals(k=0, radius2=0.01**2, view_point=[0.5, 0.5, 10.0], want_cov=True))
    assert _approx_cell_counts(cloud, info).max() > HUGE_CELL, info
    for key in ("normals", "curvature", "cov6"):
        assert np.array_equal(_bits(runs[0][key]), _bits(runs[1][key])), key
    assert np.isfinite(runs[0]["cov6"][:-1]).all()
    _report("huge cell: radius normals twice", t0)

    t0 = time.perf_counter()
    dst, _, _, T_ref = synth.icp_pair(20000, seed=14, noise=0.0)
    src = synth.apply(synth.invert(T_ref), dst[rng.integers(0, len(dst), 68000)])
    src = (src + 0.002 * rng.standard_normal(src.shape)).astype(F32)
    src = np.vstack([src, [[1e4, 1e4, 1e4]]]).astype(F32)
    max_d2 = F32(0.03**2)
    kw = dict(metric="p2p", max_iter=10, tol=0.0, max_d2=max_d2)
    want = orc.icp(dst, src, orc.BruteKnn(dst), **kw)
    for host_loop in (False, True):
        res = []
        for _ in range(2):
            s = cb.Cloud(ctx, src)
            assert _approx_cell_counts(src, s.grid_info()).max() > HUGE_CELL
            res.append(cb.Icp(ctx, cb.Cloud(ctx, dst), s).estimate(host_loop=host_loop, **kw))
        assert np.array_equal(res[0]["T"], res[1]["T"]) and res[0]["num_corr"] == res[1]["num_corr"], host_loop
        assert res[0]["num_corr"] == want["num_corr"], (host_loop, res[0]["num_corr"], want["num_corr"])
        assert frob(res[0]["T"], want["T"]) < 1e-5, (host_loop, frob(res[0]["T"], want["T"]))
    _report("huge cell: ICP twice on both loops", t0)


# ---- cell faces and bound edges --------------------------------------------------------------------------------------
def test_queries_on_cell_faces(cb, ctx, orc):
    """Queries exactly on cell faces, one ulp either side and within 2^-10 cell of them (the pruning margin), on one
    axis and on all three at once. Face positions from grid_info() and the bounding box: origin = min - h."""
    t0 = time.perf_counter()
    rng = np.random.default_rng(21)
    ref = rng.random((20000, 3), dtype=F32)
    cl = cb.Cloud(ctx, ref)
    info = cl.grid_info()
    h = float(info["cell_edge"])
    dims = info["dims"]
    assert min(dims) >= 10, info
    org = ref.astype(np.float64).min(axis=0) - h

    def face(ax, n):
        return (org[ax] + rng.integers(1, dims[ax] - 1, n) * h).astype(F32)

    def variants(f, n):
        d = h / 1024
        up, dn = np.nextafter(f, F32(np.inf)), np.nextafter(f, F32(-np.inf))
        return [f, up, dn] + [(f + s * d * rng.random(n)).astype(F32) for s in (-1, 1)] + [(f + F32(s * d)).astype(F32)
                                                                                             for s in (-1, 1)]

    parts = []
    for ax in range(3):
        for v in variants(face(ax, 300), 300):
            q = rng.random((300, 3), dtype=F32)
            q[:, ax] = v
            parts.append(q)
    corner = np.stack([face(ax, 500) for ax in range(3)], axis=1)
    parts += [corner, np.stack([np.nextafter(corner[:, ax], F32(np.inf)) for ax in range(3)], axis=1)]
    qry = np.vstack(parts).astype(F32)
    r2 = F32(0.02**2)
    _check(cb, ctx, orc, ref, qry, max_d2=FMAX, ks=(4, 16), ref=cl)
    _check(cb, ctx, orc, ref, qry, max_d2=r2, ks=(16,), r2=F32(0.03**2), corr_d2=r2, ref=cl)
    _report(f"{len(qry)} face queries (grid {info})", t0)


def test_points_exactly_on_the_bound_are_excluded(cb, ctx, orc):
    """Integer lattice references and half-integer queries: d2 of exactly 0.25, 0.5, 0.75, 1, 1.25 ... A point at d2
    equal to max_d2 / radius2 fails the strict d2 < bound test and must be left out, by every search."""
    t0 = time.perf_counter()
    rng = np.random.default_rng(22)
    g = np.arange(16, dtype=np.float64)
    ref = np.stack(np.meshgrid(g, g, g, indexing="ij"), axis=-1).reshape(-1, 3)
    ref = ref[rng.permutation(len(ref))].astype(F32)
    cl = cb.Cloud(ctx, ref)
    info = cl.grid_info()
    assert info["dims"][0] >= 10, info
    base = ref[rng.choice(len(ref), 400)].astype(np.float64)
    steps = np.array([[0, 0, 0], [0.5, 0, 0], [0.5, 0.5, 0], [0.5, 0.5, 0.5], [1, 0.5, 0], [1, 1, 0.5]])
    qry = (base[:, None, :] + steps[None, :, :]).reshape(-1, 3).astype(F32)
    for bound in (0.25, 0.5, 0.75, 1.0, 1.25):
        b = F32(bound)
        out = _check(cb, ctx, orc, ref, qry, max_d2=b, ks=(8,), r2=b, corr_d2=b, ref=cl)
        idx, d2 = out["knn1"]
        assert (d2[idx >= 0] < b).all() and (out["radius"][2] < b).all() and (out["corr"][2] < b).all()
        if bound <= 0.75:  # queries whose nearest point sits exactly on the bound found nothing
            assert (idx < 0).any()
    _report("lattice bound edges", t0)


# ---- tiny extents ----------------------------------------------------------------------------------------------------
def test_tiny_extent_cloud(cb, ctx, orc):
    """A cloud of extent 1e-30: every d2 inside it underflows to 0 (the answer is the lowest index), queries 1e-21
    away see subnormal d2, and h_safe^2 underflows, so nothing is pruned. The answers stay exact, and queries far
    outside in cell units still hand over to the block walk (far_sweep.cuh) rather than crossing 2^24 shells."""
    rng = np.random.default_rng(31)
    ref = (rng.random((20000, 3)) * 1e-30).astype(F32)
    cl = cb.Cloud(ctx, ref)
    info = cl.grid_info()
    assert info["cell_edge"] < 1e-31 and min(info["dims"]) > 3, info
    near = ref[rng.choice(len(ref), 1500)]
    far = (ref[rng.choice(len(ref), 300)] + np.array([1e-21, 0, 0])).astype(F32)
    qry = np.vstack([near, far]).astype(F32)
    q = cb.Cloud(ctx, qry)
    cb.knn1_radius(ctx, cl, q, None, FMAX)
    t0 = time.perf_counter()
    cb.knn1_radius(ctx, cl, q, None, FMAX)
    dt = time.perf_counter() - t0
    print(f"[grid-edges] tiny extent: unbounded 1-NN of {len(qry)} queries: {dt:.3f} s")
    assert dt < 5.0
    t0 = time.perf_counter()
    out = _check(cb, ctx, orc, ref, qry, max_d2=FMAX, ks=(1, 16, 17), ref=cl)
    assert (out["knn1"][0][:1500] == 0).all()  # all d2 are 0: the lowest index everywhere
    assert (out["knn1"][1][1500:] > 0).all() and (out["knn1"][1][1500:] < FMIN).all()
    _check(cb, ctx, orc, ref, far[:100], max_d2=F32(1e-40), ks=(), r2=F32(1e-40), corr_d2=F32(1e-40), ref=cl)
    _check(cb, ctx, orc, ref, near[:50], max_d2=F32(FMIN), ks=(), r2=F32(FMIN), ref=cl)
    _check_normals_k(cb, ctx, orc, ref, 8)
    _report(f"tiny extent (grid {info})", t0)
