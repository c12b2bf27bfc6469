"""Normal estimation (normals.cu, robust_normals.cu -> finish_point in normals_out.cuh -> sym3_smallest in
sym3_eigen.cuh) at its scale, neighbourhood-size and orientation edges, against float64.

Every case compares the covariance (cov6) bit for bit with the oracle's restatement over brute-force neighbourhoods
(radius mode: with a float64 covariance of the same neighbour set, within a derived bound), the NaN pattern exactly,
and every point's normal and curvature with float64 eigh of its own returned cov6 (normals_ref.check_eigen: no gap
filter, every point). The oracle's own double Jacobi stops at an absolute threshold, so its normals are not used as
the reference: eigh of the returned bits is exact input at every scale. Each test prints its worst ratios.

The cases:
  - power-of-two scale sweep (kNN, kNN-in-radius and MCD) from 2^-72 up to the scale at which the covariance
    overflows, through the scales at which the largest entry first drops below 2^-126 and 2^-128 (below which 1 / scale
    would overflow without sym3_smallest's rescaling of subnormal matrices); exact scalings keep the normal and
    curvature bits;
  - k at every kernel-template and admission edge, on clouds of 3, k - 1, k and k + 1 points with lattice ties;
  - radius neighbourhoods from fewer than 3 points to several thousand, near and far from the origin, with NaN / Inf
    points;
  - exactly coplanar, collinear, w0 = w1 and coincident neighbourhoods;
  - the orientation rules (view point, reference normals) restated in fp32;
  - the eigen step directly (tests/cuda/solve_harness.cu): subnormal, boundary, zero, NaN and Inf matrices.
"""
import os
import time

import numpy as np
import pytest

import cxx
from cilantro_b200 import synth
from normals_ref import check_eigen, fmt, merge
from oracle import robust_normals as orn

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "cilantro_b200", "csrc")
HARNESS = os.path.join(ROOT, "tests", "cuda", "solve_harness.cu")
F32 = np.float32
FMAX = float(np.finfo(F32).max)
TINY = 2.0 ** -126  # smallest normal fp32
VP = (0.5, 0.5, 10.0)


def _bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


def _report(name, worst, t0=None):
    took = f" ({time.perf_counter() - t0:.2f} s)" if t0 is not None else ""
    print(f"[normals-edges] {name}{took}: {fmt(worst)}")


def _plain(cb, ctx, orc, pts, k, r2, vp=VP, label=""):
    """cb_cloud_estimate_normals against the oracle's covariance (bit for bit, NaN pattern) and float64."""
    got = cb.Cloud(ctx, pts).estimate_normals(k=k, radius2=r2, view_point=vp, want_cov=True)
    want = orc.estimate_normals(pts, orc.BruteKnn(pts), k=k, radius2=r2 if r2 > 0 else None, view_point=vp)
    valid = want[3] >= 3
    assert np.array_equal(~np.isnan(got["cov6"]).any(axis=1), valid), label
    assert np.array_equal(_bits(got["cov6"][valid]), _bits(want[2][valid])), (label, "covariance not bit-exact")
    return got, want[3], check_eigen(got["cov6"], got["normals"], got["curvature"], label)


def _mcd(cb, ctx, pts, k, r2, vp=VP, label="", chi_square_threshold=6.25):
    """cb_cloud_estimate_normals_mcd against oracle/robust_normals.py (status and cov6 bit for bit) and float64."""
    kw = dict(num_trials=2, num_refinements=1, chi_square_threshold=chi_square_threshold, seed=3)
    got = cb.Cloud(ctx, pts).estimate_normals_mcd(k=k, radius2=r2, view_point=vp, want_cov=True, **kw)
    want = orn.estimate_normals_mcd(pts, k=k, radius2=r2, view_point=vp, **kw)
    assert np.array_equal(got["status"], want["status"]), label
    assert np.array_equal(_bits(got["cov6"]), _bits(want["cov6"])), (label, "covariance not bit-identical")
    return got, want["status"], check_eigen(got["cov6"], got["normals"], got["curvature"], label)


# ---- power-of-two scale sweep ----------------------------------------------------------------------------------------
def _sweep_clouds():
    surface, _ = synth.surface_cloud(6000, seed=31, noise=0.0003)
    rng = np.random.default_rng(32)
    centres = rng.random((3, 3))
    clustered = np.vstack([c + 0.01 * rng.standard_normal((1500, 3)) for c in centres] + [rng.random((1500, 3))])
    return {"surface": surface, "clustered": clustered.astype(F32)}


def _scaled(pts0, e):
    pts = (pts0.astype(np.float64) * 2.0 ** e).astype(F32)
    assert np.array_equal(pts.astype(np.float64), pts0.astype(np.float64) * 2.0 ** e)  # exact: no subnormal coordinate
    return pts


def _sweep_scales(cov0, overflow_e):
    """-72 .. the overflow, with the first e at which a point's largest entry drops below 2^-126 and below 2^-128."""
    big = np.abs(cov0[np.isfinite(cov0).all(axis=1)]).max(axis=1).astype(np.float64)
    big = big[big > 0]

    def first_below(t):
        e = 0
        while not (big * 4.0 ** e < t).any():
            e -= 1
        return e

    e126, e128 = first_below(TINY), first_below(2.0 ** -128)
    es = {-72, -66, -60, -40, 0, 30, 60, e126 + 1, e126, e128, e128 - 1, overflow_e - 1, overflow_e}
    return sorted(es), e126, e128


def _overflow_e(orc, pts0, k, r2_0):
    """The first e (up from 60) at which a covariance of the oracle overflows."""
    for e in range(60, 100):
        pts = _scaled(pts0, e)
        r2 = F32(min(r2_0 * 4.0 ** e, FMAX)) if r2_0 else None
        cov = orc.estimate_normals(pts, orc.BruteKnn(pts), k=k, radius2=r2)[2]
        cnt = ~np.isnan(cov).all(axis=1)
        if not np.isfinite(cov[cnt]).all():
            return e
    raise AssertionError("no overflow below 2^100")


@pytest.mark.parametrize("method", ["knn", "knn_in_radius", "mcd"])
def test_power_of_two_scale_sweep(cb, ctx, orc, method):
    """Scaling a cloud (and the view point, and the radius) by 2^e is exact: wherever a point's cov6 is exactly 4^e
    times its cov6 at e = 0, the normal and the curvature must be those of e = 0 bit for bit (the eigen step sees the
    same max-scaled matrix, or the same matrix times 2^64 below 2^-126). Two exceptions, held to the float64 bounds
    only: a largest entry of 2^126 or more, where 1 / scale is subnormal and rounds; and the curvature in the normal
    path wherever the eigenvalues w0 or w1 themselves are subnormal there (fewer bits than at e = 0). MCD runs without
    the chi-square test, whose Mahalanobis distances are not finite once the determinant underflows."""
    k = 16
    r2_0 = float(F32(0.03 ** 2)) if method == "knn_in_radius" else 0.0
    if method == "mcd":
        run = lambda p, r2, vp, lb: _mcd(cb, ctx, p, k, r2, vp, lb, chi_square_threshold=-1.0)  # noqa: E731
    else:
        run = lambda p, r2, vp, lb: _plain(cb, ctx, orc, p, k, r2, vp, lb)  # noqa: E731
    total = {}
    for name, pts0 in _sweep_clouds().items():
        got0, _, _ = run(pts0, r2_0, VP, f"{method} {name} e=0")
        cov0 = got0["cov6"].astype(np.float64)
        e_over = _overflow_e(orc, pts0, k, r2_0)
        scales, e126, e128 = _sweep_scales(got0["cov6"], e_over)
        assert e128 < e126 < 0
        print(f"[normals-edges] {method} {name}: first e below 2^-126 {e126}, below 2^-128 {e128}, overflow {e_over}")
        subnormal_exact = subnormal = 0
        for e in scales:
            t0 = time.perf_counter()
            pts = _scaled(pts0, e)
            vp = tuple(float(F32(v * 2.0 ** e)) for v in VP)
            r2 = float(F32(min(max(r2_0 * 4.0 ** e, 2.0 ** -149), FMAX))) if r2_0 else 0.0
            label = f"{method} {name} e={e}"
            got, _, worst = run(pts, r2, vp, label)
            cov = got["cov6"].astype(np.float64)
            fin = np.isfinite(cov).all(axis=1)
            big = np.abs(np.where(fin[:, None], cov, 0.0)).max(axis=1)
            exact = fin & np.all(cov == cov0 * 4.0 ** e, axis=1) & (big < 2.0 ** 126)
            assert np.array_equal(_bits(got["normals"][exact]), _bits(got0["normals"][exact])), (label, "normal bits")
            # the curvature: the rescaled path, or normal-range eigenvalues (w1 >= w0 >= curv0 * trace / (1 + 1e-6))
            c0 = got0["curvature"].astype(np.float64)
            trace = cov[:, 0] + cov[:, 3] + cov[:, 5]
            with np.errstate(invalid="ignore"):
                keep = exact & ((big < TINY) | ((c0 > 0) & (c0 * trace >= 2.0 ** -125)))
            assert np.array_equal(_bits(got["curvature"][keep]), _bits(got0["curvature"][keep])), (label, "curvature")
            sub = fin & (big > 0) & (big < TINY)
            subnormal += int(sub.sum())
            subnormal_exact += int((sub & exact).sum())
            if e == e_over and method != "mcd":  # the covariance overflowed: NaN normal and curvature (check_eigen)
                assert worst["non-finite"] > int(np.isnan(cov0).any(axis=1).sum()), (label, "no overflow")
            worst = dict(worst, bit_exact=int(exact.sum()), curvature_bit_exact=int(keep.sum()), subnormal=int(sub.sum()))
            _report(label, worst, t0)
            merge(total, worst)
        assert subnormal > 0, (label, "the subnormal range was not reached")
        # (covariances summed in the subnormal range rarely scale exactly; test_sym3_subnormal_and_boundary pins the
        # bit identity of exact scalings directly)
        print(f"[normals-edges] {method} {name}: {subnormal} subnormal-range covariances, {subnormal_exact} exact")
    _report(f"scale sweep {method}, all", total)


# ---- k at every template and admission edge --------------------------------------------------------------------------
K_EDGES = (1, 2, 3, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128)
STEP = 0.25  # lattice step: every lattice d2 is an exact multiple of 1/16
R2_LATTICE = 2 * STEP ** 2  # the face diagonal: lattice neighbours at exactly radius2


def _lattice_cloud(n, seed):
    """n points: the first half on a 4 x 4 x 4 lattice (ties at every distance), the rest random in its box."""
    g = np.stack(np.meshgrid(*[np.arange(4)] * 3, indexing="ij"), axis=-1).reshape(-1, 3) * STEP
    rng = np.random.default_rng(seed)
    m = min((n + 1) // 2, len(g))
    lat = g[rng.permutation(len(g))[:m]]
    return np.vstack([lat, rng.random((n - m, 3)) * 3 * STEP]).astype(F32)


@pytest.mark.parametrize("mode", ["knn", "knn_in_radius"])
@pytest.mark.parametrize("k", K_EDGES)
def test_k_edges(cb, ctx, orc, k, mode):
    """normals_knn_kernel<K> for the smallest K in {8, 16, 32, 64, 128} >= k, on clouds of 3, k - 1, k, k + 1 points
    and one of 700 (full lists, exact ties on the k-th slot). k <= 2 can never reach the minimum of 3 samples."""
    r2 = R2_LATTICE if mode == "knn_in_radius" else 0.0
    total = {}
    for n in sorted({3, k - 1, k, k + 1, 700} - {0}):
        pts = _lattice_cloud(n, seed=1000 * k + n)
        got, cnt, worst = _plain(cb, ctx, orc, pts, k, r2, label=f"k={k} {mode} n={n}")
        merge(total, worst)
        if k <= 2:
            assert np.isnan(got["normals"]).all() and np.isnan(got["curvature"]).all() and np.isnan(got["cov6"]).all()
        if r2:  # admission is strict: lattice neighbours at exactly radius2 are out
            d = pts[:, None, :] - pts[None, :, :]  # contract_d2 in fp32: ((dx dx) + dy dy) + dz dz
            d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
            want = np.minimum((d2 < r2).sum(axis=1), k)
            assert np.array_equal(cnt, want), (k, n)
            if n >= 64:
                assert (d2 == F32(r2)).any()
    _report(f"k={k} {mode}", total)


def test_k_above_128_rejected(cb, ctx):
    cloud = cb.Cloud(ctx, _lattice_cloud(300, seed=5))
    with pytest.raises(cb.CbError, match="error -5"):
        cloud.estimate_normals(k=129)
    with pytest.raises(cb.CbError, match="error -5"):
        cloud.estimate_normals(k=129, radius2=1.0)
    assert not np.isnan(cloud.estimate_normals(k=128)["normals"]).any()  # the context is still usable


# ---- radius mode -----------------------------------------------------------------------------------------------------
def _gamma(m):
    u = 2.0 ** -24
    return m * u / (1 - m * u)


def _radius_bound(nbr):
    """A bound on |cov_fp32 - cov_64| for the radius kernel's arithmetic over the neighbour set nbr (m x 3, in any
    summation order): fp32 mean mu' = fl(fl(1/m) fl(sum p)) is within delta = gamma_{m+1} sum|p| / m of the mean mu;
    with e = p - mu', sum e_a e_b = sum d_a d_b + m delta_a delta_b (d = p - mu: the cross terms vanish); the
    differences, products, m-term sum and the 1/(m-1) scaling add gamma_{m+4} sum|e_a e_b| / (m-1)."""
    m = len(nbr)
    p = nbr.astype(np.float64)
    delta = _gamma(m + 1) * np.abs(p).sum(axis=0) / m
    d = np.abs(p - p.mean(axis=0)) + delta
    pairs = [(0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)]
    return np.array([(m * delta[a] * delta[b] + _gamma(m + 4) * (d[:, a] * d[:, b]).sum()) / (m - 1)
                     for a, b in pairs])


def _cov64(nbr):
    p = nbr.astype(np.float64)
    d = p - p.mean(axis=0)
    C = d.T @ d / (len(p) - 1)
    return C[[0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]


def _radius_scene(offset, seed):
    """A dense blob (thousands of neighbours), a sparse sheet (tens), isolated points and pairs (fewer than 3), NaN
    and Inf points."""
    rng = np.random.default_rng(seed)
    blob = 0.02 * rng.standard_normal((5000, 3))
    sheet = np.column_stack([rng.random((3000, 2)) * 2 + 0.5, 0.001 * rng.standard_normal(3000)])
    lone = np.array([[-3.0, 0, 0], [3.0, 3, 3], [3.001, 3, 3], [-3, -3, -3], [-3, -3, -3.001], [-3, -3.001, -3]])
    pts = np.vstack([blob, sheet, lone]) + np.asarray(offset)
    bad = np.array([[np.nan, 0, 0], [0, np.inf, 0], [-np.inf, 1, 1], [np.nan] * 3, [np.inf] * 3])
    return np.vstack([pts, bad, offset + np.array([[0.0, 0.0, 0.0]])]).astype(F32)


@pytest.mark.parametrize("offset", [(0.0, 0.0, 0.0), (6.0, -10.0, 4.0)])
def test_radius_mode(cb, ctx, orc, offset):
    pts = _radius_scene(np.asarray(offset), seed=41)
    n = len(pts)
    r2 = float(F32(0.05 ** 2))
    t0 = time.perf_counter()
    cloud = cb.Cloud(ctx, pts)
    got = cloud.estimate_normals(k=0, radius2=r2, view_point=VP, want_cov=True)
    again = cloud.estimate_normals(k=0, radius2=r2, view_point=VP, want_cov=True)
    for key in ("normals", "curvature", "cov6"):
        assert np.array_equal(_bits(got[key]), _bits(again[key])), key  # repeatable bit for bit
    finite = np.isfinite(pts).all(axis=1)
    brute = orc.BruteKnn(pts)
    _, _, cnt = brute.neighborhoods(pts, 0, r2, stride=1)
    assert cnt.max() > 2000 and (cnt[finite] < 3).any() and ((cnt > 3) & (cnt < 100)).any(), (cnt.max(),)
    assert (cnt[~finite] == 0).all()
    valid = cnt >= 3
    assert np.array_equal(~np.isnan(got["cov6"]).any(axis=1), valid)
    worst = check_eigen(got["cov6"], got["normals"], got["curvature"], f"radius {offset}")
    # the covariance against float64 of the same neighbour set, in chunks (the sets hold up to several thousand)
    q = np.flatnonzero(valid)
    ratio, rel = 0.0, 0.0
    for s in range(0, len(q), 256):
        qs = q[s:s + 256]
        idx, _, c = brute.neighborhoods(pts[qs], 0, r2, stride=int(cnt[qs].max()))
        for row, i in enumerate(qs):
            nb = idx[row, :c[row]]
            assert finite[nb].all()  # NaN and Inf points are in nobody's neighbourhood
            ref, bound = _cov64(pts[nb]), _radius_bound(pts[nb])
            err = np.abs(got["cov6"][i].astype(np.float64) - ref)
            assert np.all(err <= bound), (i, c[row], err, bound)
            ratio = max(ratio, float((err / bound).max()))
            rel = max(rel, float(err.max() / np.abs(ref).max()))
    worst = dict(worst, **{"cov err/bound": ratio, "cov err/max|cov|": rel, "max count": int(cnt.max())})
    _report(f"radius mode, offset {offset}", worst, t0)


# ---- degenerate neighbourhoods ---------------------------------------------------------------------------------------
def _degenerate_sets():
    """Sets of 32 points on a dyadic grid: over the whole set or 16 of it the mean (1/32, 1/16) and every sum of the
    covariance are exact, only the final 1 / (m - 1) rounds."""
    rng = np.random.default_rng(51)
    q = lambda a: np.round(np.asarray(a) * 64) / 64  # noqa: E731
    xy = q(rng.random((32, 2)))
    out = {"coplanar z = c": np.column_stack([xy, np.full(32, 0.375)])}
    out["coplanar x + y + z = 1"] = np.column_stack([xy, 1.0 - xy[:, 0] - xy[:, 1]])
    out["coplanar x = y"] = np.column_stack([xy[:, 0], xy[:, 0], xy[:, 1]])
    t = np.arange(-16, 16)[:, None] / 64.0
    out["collinear (1, 2, 3)"] = t * np.array([1.0, 2.0, 3.0]) + 0.5
    out["collinear x"] = np.column_stack([t[:, 0], np.full(32, 0.25), np.full(32, -0.5)])
    base = q(rng.random((8, 3)) - 0.5) * [1.0, 1.0, 3.0]
    rot = [base, base[:, [1, 0, 2]] * [-1, 1, 1], base * [-1, -1, 1], base[:, [1, 0, 2]] * [1, -1, 1]]
    out["w0 = w1 (four-fold about z)"] = np.vstack(rot)  # cov = diag(a, a, c), c > a
    return {k: v.astype(F32) for k, v in out.items()}


def test_degenerate_neighbourhoods(cb, ctx, orc):
    total = {}
    for name, pts in _degenerate_sets().items():
        for k in (len(pts), 16):  # the whole set, and half of it
            got, _, worst = _plain(cb, ctx, orc, pts, k, 0.0, label=f"{name} k={k}")
            merge(total, worst)
            if k == len(pts):
                C = got["cov6"].astype(np.float64)
                if name.startswith("coplanar z") or name.startswith("collinear x"):
                    assert (C[:, [2, 4, 5]] == 0).all()  # exact: the eigen step sees an exact zero eigenvalue
                if name.startswith("w0 = w1"):
                    assert (C[:, 0] == C[:, 3]).all() and (C[:, [1, 2, 4]] == 0).all() and (C[:, 5] > C[:, 0]).all()
        _report(name, worst)
    # >= k coincident copies: a zero covariance, the normal +-e_x, a NaN curvature; the view point decides the sign
    rng = np.random.default_rng(52)
    p = np.float32([0.375, -0.25, 0.625])  # few mantissa bits: the fp32 mean of the copies is exact
    pts = np.vstack([np.tile(p, (20, 1)), rng.random((200, 3)) + 2]).astype(F32)
    for vp, sign in ((None, 1.0), ((5.0, 0.0, 0.0), 1.0), ((-5.0, 0.0, 0.0), -1.0)):
        got, _, worst = _plain(cb, ctx, orc, pts, 16, 0.0, vp=vp, label=f"coincident vp={vp}")
        assert (got["cov6"][:20] == 0).all()
        assert np.array_equal(got["normals"][:20], np.tile(np.float32([sign, 0, 0]), (20, 1)))
        assert np.isnan(got["curvature"][:20]).all()
        assert worst["zero"] == 20
    _report("degenerate, all", total)


# ---- orientation -----------------------------------------------------------------------------------------------------
def _dot32(n, e):
    """finish_point's fp32 dot: n0 e0 + (n1 e1 + n2 e2), one rounding per operation."""
    n, e = np.asarray(n, F32), np.asarray(e, F32)
    return n[:, 0] * e[:, 0] + (n[:, 1] * e[:, 1] + n[:, 2] * e[:, 2])


def _flip(n, d):
    return np.where((d < 0)[:, None], -n, n)


def test_orientation_edges(cb, ctx):
    pts, _ = synth.surface_cloud(4000, seed=61, noise=0.0005)
    n0 = cb.Cloud(ctx, pts).estimate_normals(k=12)["normals"]  # unoriented: the eigenvector as solved
    assert not np.isnan(n0).any()
    # a view point with a NaN or Inf component is no view point (view_point_.allFinite())
    for vp in ((np.nan, 0.5, 10.0), (0.5, np.inf, 10.0), (0.5, 0.5, -np.inf)):
        got = cb.Cloud(ctx, pts).estimate_normals(k=12, view_point=vp)["normals"]
        assert np.array_equal(_bits(got), _bits(n0)), vp
    # view points: far, and exactly on cloud points (e = 0 there: d = 0, not < 0, so unflipped)
    for j in (0, 1234, 3999):
        vp = pts[j].copy()
        got = cb.Cloud(ctx, pts).estimate_normals(k=12, view_point=vp)["normals"]
        want = _flip(n0, _dot32(n0, vp[None, :] - pts))
        assert np.array_equal(_bits(got), _bits(want)), j
        assert np.array_equal(_bits(got[j]), _bits(n0[j]))
    # reference normals: NaN or zero rows leave the normal as solved; they take precedence over the view point
    rng = np.random.default_rng(62)
    ref = rng.standard_normal(pts.shape).astype(F32)
    ref[::7] = np.nan
    ref[3::7] = 0.0
    ref[5::7, 1] = np.nan
    ref[6::7] = -0.0
    for vp in (None, (0.5, 0.5, 10.0), (0.5, 0.5, -10.0)):
        got = cb.Cloud(ctx, pts, ref).estimate_normals(k=12, view_point=vp, use_current_as_ref=True)["normals"]
        d = _dot32(n0, ref)
        want = _flip(n0, d)
        assert np.array_equal(_bits(got), _bits(want)), vp
        assert np.array_equal(_bits(got[~(d < 0)]), _bits(n0[~(d < 0)]))
    flipped = (_dot32(n0, ref) < 0).sum()
    assert 0 < flipped < len(pts)
    print(f"[normals-edges] orientation: {flipped} of {len(pts)} normals flipped by the reference normals")


# ---- the eigen step directly -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sym3_exe(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("sym3_edges") / "solve_harness_dev")
    return cxx.harness(HARNESS, exe, [f"-I{CSRC}"], device=True)


def _sym3(exe, cases, tmpdir):
    src, dst = os.path.join(tmpdir, "sym3.in"), os.path.join(tmpdir, "sym3.out")
    np.ascontiguousarray(cases, F32).tofile(src)
    cxx.run(exe, "sym3", src, dst)
    out = np.fromfile(dst, F32).reshape(-1, 7)
    return out[:, :3], out[:, 3:6], out[:, 6]


def _grid_cov(rng, spectrum):
    """A covariance with the given spectrum, rotated, its largest |entry| exactly 1 and every entry a multiple of
    2^-12 (so that any 2^-k scaling with k <= 137 is exact in fp32)."""
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    C = q @ np.diag(spectrum) @ q.T
    c = C[[0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
    c = np.round(c / np.abs(c).max() * 4096) / 4096
    return c.astype(F32)


def test_sym3_subnormal_and_boundary(sym3_exe, tmp_path):
    rng = np.random.default_rng(71)
    base = [_grid_cov(rng, s) for s in ([0.05, 0.3, 1.0], [1e-3, 0.2, 1.0], [0.0, 0.4, 1.0], [0.5, 0.5, 1.0],
                                         [0.0, 0.0, 1.0], [0.2, 0.7, 0.9]) for _ in range(4)]
    cases, kinds, pairs = [], [], []  # pairs: (case index, index of the normal-range matrix it scales exactly)

    def add(c, kind, of=None):
        cases.append(np.asarray(c, F32))
        kinds.append(kind)
        if of is not None:
            pairs.append((len(cases) - 1, of))

    for b in base:
        add(b, "normal range")
        i0 = len(cases) - 1
        for kk in (127, 128, 129, 131, 134, 137):  # exact 2^-k scalings, every entry subnormal or zero
            s = (b.astype(np.float64) * 2.0 ** -kk).astype(F32)
            assert np.array_equal(s.astype(np.float64), b.astype(np.float64) * 2.0 ** -kk)
            add(s, f"2^-{kk} scaled", of=i0)
        for t in (-126, -128):  # the largest entry exactly at 2^t and one ulp either side
            s = (b.astype(np.float64) * 2.0 ** t).astype(F32)
            big = int(np.argmax(np.abs(s)))
            for v in (np.nextafter(s[big], F32(0)), s[big], np.nextafter(s[big], F32(np.inf) * np.sign(s[big]))):
                c = s.copy()
                c[big] = v
                add(c, f"largest at 2^{t} (+-1 ulp)", of=i0 if v == s[big] and t == -128 else None)
    ts = float(np.finfo(F32).smallest_subnormal)
    for c in ([ts, 0, 0, 0, 0, 0], [0, 0, 0, ts, 0, ts], [ts] * 6, [0, ts, 0, 0, 0, 0], [ts, -ts, 0, ts, 0, 0]):
        add(np.asarray(c), "smallest subnormal")
    for _ in range(12):  # zeros mixed with small integers times 2^-149: exact scalings of the integer matrices
        A = rng.integers(-2, 3, (3, 3)) * (rng.random((3, 3)) < 0.5)
        M = A @ A.T  # positive semi-definite, like a covariance
        m = M[[0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
        if not m.any():
            m[0] = 1
        add(m, "small integers")
        add(m * ts, "small integers times 2^-149", of=len(cases) - 1)
    add(np.zeros(6), "zero")
    special = []
    for j in range(6):
        for v in (np.inf, -np.inf, np.nan):
            c = base[0].copy()
            c[j] = v
            special.append(len(cases))
            add(c, "non-finite entry")
    special.append(len(cases))
    add(np.full(6, np.nan), "all NaN")
    special.append(len(cases))
    add(np.full(6, np.inf), "all Inf")

    w, n, curv = _sym3(sym3_exe, np.array(cases), str(tmp_path))
    for i in special:  # NaN throughout
        assert np.isnan(w[i]).all() and np.isnan(n[i]).all() and np.isnan(curv[i]), (kinds[i], cases[i], w[i], n[i])
    z = kinds.index("zero")
    assert (w[z] == 0).all() and np.array_equal(n[z], F32([1, 0, 0])) and np.isnan(curv[z])
    for i, i0 in pairs:  # exact scalings: the normal and the curvature bit for bit
        assert np.array_equal(_bits(n[i]), _bits(n[i0])), (kinds[i], cases[i0], n[i], n[i0])
        assert np.array_equal(_bits(curv[i]), _bits(curv[i0])), (kinds[i], cases[i0], curv[i], curv[i0])
    keep = np.array([i for i in range(len(cases)) if i not in special and kinds[i] != "zero"])
    worst = {}
    for kind in sorted(set(kinds[i] for i in keep)):
        sel = np.array([i for i in keep if kinds[i] == kind])
        worst[kind] = check_eigen(np.array(cases)[sel], n[sel], curv[sel], kind)
        # eigenvalues: w2 within 1e-6 relative, all within 1e-6 w2 absolute (plus the subnormal spacing of fp32)
        wr = np.linalg.eigvalsh(np.array([[[c[0], c[1], c[2]], [c[1], c[3], c[4]], [c[2], c[4], c[5]]]
                                          for c in np.array(cases, np.float64)[sel]]))
        err = np.abs(w[sel].astype(np.float64) - wr).max(axis=1)
        scale = np.abs(wr).max(axis=1)
        assert np.all(err <= 1e-6 * scale + 2.0 ** -149), (kind, err / scale)
        _report(f"sym3 {kind}", worst[kind])
    assert len(pairs) > 150
