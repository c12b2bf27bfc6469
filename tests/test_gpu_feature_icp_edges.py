"""Feature-space correspondence search of the rigid ICP on the device (cb_icp_set_features, feature_search.cu) against
an exact restatement of the same search (tests/feature_search_ref.py, itself pinned to the brute-force oracle by
test_feature_search_ref.py), per query: the index and the value bits of every source query's match (second_to_first)
and of every destination query's match (first_to_second, over the grid rebuilt around the moved source with rotated
tails). Beyond the textured-sheet scene of test_gpu_feature_icp.py: clouds larger than one and two grid-stride passes,
colour weights from 2^-70 to 1e20, a scene whose feature-nearest points lie far beyond the shell walk's reach (the far
sweep, which must not use its xyz radius bound), exact ties on a dyadic lattice, large rotations, offsets and scales,
non-finite xyz, degenerate geometry, and a 30-iteration loop at scale against the oracle's ICP."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

import feature_search_ref as fsr
from cilantro_b200 import capi, synth
from conftest import frob

pytestmark = pytest.mark.gpu

FLT_MAX = float(np.finfo(np.float32).max)
KINDS = ["point_normal", "point_color", "point_normal_color"]
DIRS = {"s2f": "second_to_first", "f2s": "first_to_second"}
W_N, W_C = 0.5, 5.0
I34 = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)
T0 = np.array([[0.9998, -0.0175, 0.0, 0.025], [0.0175, 0.9998, 0.0, -0.015], [0.0, 0.0, 1.0, 0.0005]], np.float32)


@pytest.fixture(scope="module")
def F(orc):
    from oracle import feature_icp

    return feature_icp


def _rigid(axis, angle, t=(0.0, 0.0, 0.0), centre=(0.0, 0.0, 0.0)):
    """Rotation by angle about axis through centre, then translation t: a 3x4 float32 transform."""
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    R = np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K
    c = np.asarray(centre, np.float64)
    return np.hstack([R, (c - R @ c + np.asarray(t, np.float64))[:, None]]).astype(np.float32)


def _arrays(kind, s):
    nrm, col = "normal" in kind, "color" in kind
    return dict(dst_normals=s["dst_normals"] if nrm else None, dst_colors=s["dst_colors"] if col else None,
                src_normals=s["src_normals"] if nrm else None, src_colors=s["src_colors"] if col else None)


class Search:
    """One scene, one feature kind and weights: the device's per-query answers and the restatement's."""

    def __init__(self, ctx, F, kind, s, w_n=W_N, w_c=W_C):
        self.F, self.kind, self.s = F, kind, s
        a = _arrays(kind, s)
        self.dt = F.tails(kind, a["dst_normals"], a["dst_colors"], w_n, w_c)
        self.st = F.tails(kind, a["src_normals"], a["src_colors"], w_n, w_c)
        self.icp = capi.Icp(ctx, capi.Cloud(ctx, s["dst"]), capi.Cloud(ctx, s["src"]))
        self.icp.set_features(kind, normal_weight=w_n, color_weight=w_c, **a)

    def device_list(self, T, max_d2, d):
        self.icp.estimate(metric="p2p", max_iter=1, tol=0.0, T_init=T, max_d2=max_d2, search_dir=DIRS[d])
        return self.icp.correspondences()

    def device(self, T, max_d2, d):
        f, sec, v = self.device_list(T, max_d2, d)
        n = self.s["src"].shape[0] if d == "s2f" else self.s["dst"].shape[0]
        return fsr.per_query(f, sec, v, n, by="second" if d == "s2f" else "first")

    def features(self, T):
        return np.hstack([self.s["dst"], self.dt]), self.F.features(self.kind, T, self.s["src"], self.st)

    def expected(self, T, max_d2, d):
        dst_f, src_f = self.features(T)
        return fsr.knn1(dst_f, src_f, max_d2) if d == "s2f" else fsr.knn1(src_f, dst_f, max_d2)

    def oracle_list(self, T, max_d2, d):
        return self.F.engine_correspondences(self.kind, self.s["dst"], self.dt, self.s["src"], self.st, T, max_d2,
                                             search_dir=DIRS[d])


def _bounded(want, r):
    """The answer under the radius r from the unbounded one: the nearest point if its d2 < r, else none."""
    ok = want[1] < np.float32(r)
    return np.where(ok, want[0], -1), np.where(ok, want[1], np.float32(r))


def _attained(want):
    """A radius equal to an attained distance (the median one), so that the strict d2 < max_d2 is hit exactly."""
    hit = want[1][want[0] >= 0]
    return float(np.sort(hit)[hit.size // 2])


def _check(got, want, what):
    gi, gd = got
    wi, wd = want
    bad = np.flatnonzero(gi != wi)
    assert bad.size == 0, (what, bad.size, bad[:5], gi[bad[:5]], wi[bad[:5]], gd[bad[:5]], wd[bad[:5]])
    m = wi >= 0
    assert m.any(), what
    bad = np.flatnonzero(gd[m].view(np.uint32) != wd[m].view(np.uint32))
    assert bad.size == 0, (what, bad.size, gd[m][bad[:5]], wd[m][bad[:5]])


def _check_all(S, T, dirs=("s2f", "f2s"), radii=("attained", FLT_MAX), lists=False, tag=""):
    """Per query against the restatement for each direction and radius; with lists=True the whole list (order
    included) against the oracle's engine too."""
    for d in dirs:
        unbounded = S.expected(T, FLT_MAX, d)
        for r in radii:
            r = _attained(unbounded) if r == "attained" else r
            want = _bounded(unbounded, r)
            what = (tag, S.kind, d, r)
            _check(S.device(T, r, d), want, what)
            if lists:
                got, ref = S.device_list(T, r, d), S.oracle_list(T, r, d)
                assert all(np.array_equal(x, y) for x, y in zip(got[:2], ref[:2])), what
                assert np.array_equal(got[2].view(np.uint32), ref[2].view(np.uint32)), what


# ------------------------------------------------------------------------------------------------------- weight sweep


@pytest.mark.parametrize("kind", ["point_color", "point_normal_color"])
@pytest.mark.parametrize("w_c", [2.0 ** -70, 1e-3, 5.0, 1e3, 1e20])
def test_colour_weight_sweep(ctx, F, kind, w_c):
    """At 2^-70 the colour squares are subnormal or zero; at 1e20 a colour square is +inf unless the colours agree to
    within ~0.18 / 1e20 * sqrt(FLT_MAX)."""
    s = synth.textured_sheet_pair(20000, seed=21)
    S = Search(ctx, F, kind, s, w_c=w_c)
    _check_all(S, T0, tag=w_c)
    if w_c == 1e20:
        _, src_f = S.features(T0)
        dst_f = np.hstack([s["dst"], S.dt])
        d = fsr.feature_d2(src_f[:200, None, :], dst_f[None, :2000, :])
        assert np.isinf(d).mean() > 0.5  # most pairs are at +inf: only near-equal colours are at a finite distance


def _far_scene(n, seed):
    """Colour = position in the unit cube; each source point carries the colour of the position half the extent away
    along every axis (wrapped), so with a large colour weight its feature-nearest destination point is ~0.87 away."""
    rng = np.random.default_rng(seed)
    dst, src = rng.random((n, 3)), rng.random((n, 3))
    nrm = lambda m: (lambda v: v / np.linalg.norm(v, axis=1, keepdims=True))(rng.normal(size=(m, 3)))  # noqa: E731
    f = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731
    return dict(dst=f(dst), dst_colors=f(dst), dst_normals=f(nrm(n)), src=f(src), src_colors=f((src + 0.5) % 1.0),
                src_normals=f(nrm(n)))


@pytest.mark.parametrize("kind", ["point_color", "point_normal_color"])
def test_feature_nearest_far_beyond_the_shell_walk(ctx, F, kind):
    """The shell walk spends its row budget long before it reaches the match and restarts on the far sweep. There the
    xyz radius bound (the far corner of the xyz-nearest non-empty block) would cut the match off: the search must run
    the sweep without it."""
    n = 150_000
    s = _far_scene(n, seed=31)
    S = Search(ctx, F, kind, s, w_c=1e3)
    _check_all(S, T0, tag="far")
    # the scene does what it is for: the feature-nearest point is not the xyz-nearest one, and for most queries it lies
    # beyond any block that holds the xyz-nearest point (cell edge h as the grid picks it for a uniform cube)
    dst_f, src_f = S.features(T0)
    want = fsr.knn1(dst_f, src_f, FLT_MAX)[0]
    q = src_f[:, :3].astype(np.float64)
    dx, ix = cKDTree(s["dst"].astype(np.float64)).query(q, workers=-1)
    h = 1.0 / np.ceil(np.cbrt(n / 2.0))
    df = np.linalg.norm(q - s["dst"][want], axis=1)
    assert (want != ix).mean() > 0.9
    beyond = (df > dx + 16 * np.sqrt(3) * h).mean()
    assert beyond > 0.5, beyond


# ------------------------------------------------------------------------------------------------------- exact ties


@pytest.mark.parametrize("kind", KINDS)
def test_exact_ties_go_to_the_lowest_index(ctx, F, kind):
    """Dyadic lattice, duplicated points, palette colours, queries at lattice midpoints: every feature distance is exact,
    most answers are a tie between several points, and the answer is the lowest index in both directions."""
    s = fsr.lattice_scene(4000, 4000, seed=41)
    S = Search(ctx, F, kind, s, w_n=0.5, w_c=1.0)
    for T in (I34, _rigid((0, 0, 1), 0.0, t=(0.25, -0.125, 0.5))):  # a dyadic translation keeps every value exact
        _check_all(S, T, lists=True, tag="ties")
    dst_f, src_f = S.features(I34)
    best = fsr.knn1(dst_f, src_f, FLT_MAX)[1]
    tied = tail_zero_tie = 0
    for i in range(0, src_f.shape[0], 256):
        d = fsr.feature_d2(src_f[i:i + 256, None, :], dst_f[None, :, :])
        at = d == best[i:i + 256, None]
        tied += int((at.sum(1) > 1).sum())
        # a candidate at xyz distance == best with a zero tail difference tied with one that has a tail term
        xyz = fsr.feature_d2(src_f[i:i + 256, None, :3], dst_f[None, :, :3])
        pure = (at & (xyz == d)).any(1) & (at & (xyz < d)).any(1)
        tail_zero_tie += int(pure.sum())
    assert tied > 0.4 * src_f.shape[0], tied
    if "color" in kind:  # (unit normals at w_n = 0.5 never tie with a pure xyz distance on this lattice)
        assert tail_zero_tie > 50, tail_zero_tie


# ---------------------------------------------------------------------------------------- rotations, offsets, scales


ROTATIONS = {
    "90_z": _rigid((0, 0, 1), np.pi / 2, centre=(0.5, 0.5, 0.0)),
    "180_xy": _rigid((1, 1, 0), np.pi, centre=(0.5, 0.5, 0.0)),
    "2.5rad": _rigid((0.3, -0.5, 0.8), 2.5, t=(0.4, -0.2, 0.3)),
}


@pytest.mark.parametrize("kind", ["point_normal", "point_normal_color"])
@pytest.mark.parametrize("rot", list(ROTATIONS))
def test_large_rotations(ctx, F, kind, rot):
    """s2f rotates the query normals, f2s the normals gathered into the moved source's grid."""
    s = synth.textured_sheet_pair(5000, seed=51)
    _check_all(Search(ctx, F, kind, s), ROTATIONS[rot], lists=True, tag=rot)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("scale,offset", [(1.0, 1e4), (1e-3, 0.0), (1e3, 0.0)])
def test_offsets_and_scales(ctx, F, kind, scale, offset):
    """xyz scaled and moved, tails unchanged: the balance between the xyz and the tail terms moves by scale^2."""
    s = synth.textured_sheet_pair(5000, seed=61)
    for key in ("dst", "src"):
        s[key] = (s[key].astype(np.float64) * scale + offset).astype(np.float32)
    c = np.full(3, 0.5 * scale + offset)
    T = _rigid((0, 0, 1), 0.0175, t=(0.025 * scale, -0.015 * scale, 0.0), centre=c)
    _check_all(Search(ctx, F, kind, s), T, lists=True, tag=(scale, offset))


# ------------------------------------------------------------------------------------------------ input edges


@pytest.mark.parametrize("kind", KINDS)
def test_non_finite_xyz_never_match(ctx, F, kind):
    s = synth.textured_sheet_pair(5000, seed=71)
    rng = np.random.default_rng(71)
    bad = {}
    for key in ("dst", "src"):
        rows = rng.choice(5000, 60, replace=False)
        s[key][rows[:20], 0] = np.nan
        s[key][rows[20:40], 1] = np.inf
        s[key][rows[40:], 2] = -np.inf
        bad[key] = rows
    S = Search(ctx, F, kind, s)
    _check_all(S, T0, lists=True, tag="non-finite")
    for d in ("s2f", "f2s"):
        f, sec, _ = S.device_list(T0, FLT_MAX, d)
        assert len(f) > 4000
        assert not np.isin(f, bad["dst"]).any() and not np.isin(sec, bad["src"]).any()
    # the finite rows get the answer of the search over the finite rows alone
    keep_d = np.setdiff1d(np.arange(5000), bad["dst"])
    keep_s = np.setdiff1d(np.arange(5000), bad["src"])
    dst_f, src_f = S.features(T0)
    sub = S.F.knn1(dst_f[keep_d], src_f[keep_s], FLT_MAX)
    got = S.device(T0, FLT_MAX, "s2f")
    assert np.array_equal(got[0][keep_s], keep_d[sub[0]])
    assert np.array_equal(got[1][keep_s].view(np.uint32), sub[1].view(np.uint32))


def _one_point_scene(n, seed):
    """Every destination point at one xyz with its own colour: a pure colour search inside one cell."""
    rng = np.random.default_rng(seed)
    f = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731
    nrm = rng.normal(size=(2 * n, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    return dict(dst=f(np.tile([[0.3, -0.2, 0.7]], (n, 1))), dst_colors=f(rng.random((n, 3))), dst_normals=f(nrm[:n]),
                src=f(np.array([0.3, -0.2, 0.7]) + 0.01 * rng.normal(size=(n, 3))), src_colors=f(rng.random((n, 3))),
                src_normals=f(nrm[n:]))


def _colinear_scene(n, seed):
    rng = np.random.default_rng(seed)
    f = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731
    line = lambda t: np.outer(t, [1.0, 2.0, -1.0]) + [0.1, 0.2, 0.3]  # noqa: E731
    nrm = rng.normal(size=(2 * n, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    td, ts = rng.random(n), rng.random(n)
    return dict(dst=f(line(td)), dst_colors=f(np.stack([td, td ** 2, 1 - td], 1)), dst_normals=f(nrm[:n]),
                src=f(line(ts)), src_colors=f(np.stack([ts, ts ** 2, 1 - ts], 1) + 0.05 * rng.random((n, 3))),
                src_normals=f(nrm[n:]))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("scene", ["one_point", "colinear"])
def test_degenerate_geometry(ctx, F, kind, scene):
    s = (_one_point_scene if scene == "one_point" else _colinear_scene)(3000, seed=81)
    _check_all(Search(ctx, F, kind, s), T0 if scene == "colinear" else I34, lists=True, tag=scene)


# ---------------------------------------------------------------------------------------------------- the loop


def test_loop_at_scale_with_a_large_colour_weight(ctx, F):
    s = synth.textured_sheet_pair(20000, seed=91)
    kind = "point_normal_color"
    kw = dict(metric="combined", w_pt=0.1, w_pl=1.0, max_iter=30, tol=0.0, max_d2=1.0, search_dir="both")
    a = _arrays(kind, s)
    dt = F.tails(kind, a["dst_normals"], a["dst_colors"], W_N, 50.0)
    st = F.tails(kind, a["src_normals"], a["src_colors"], W_N, 50.0)
    icp = capi.Icp(ctx, capi.Cloud(ctx, s["dst"], s["dst_normals"]), capi.Cloud(ctx, s["src"]))
    icp.set_features(kind, normal_weight=W_N, color_weight=50.0, **a)
    got = icp.estimate(**kw)
    want = F.icp(kind, s["dst"], dt, s["src"], st, dst_n=s["dst_normals"], **kw)
    assert got["iterations"] == want["iterations"] == 30
    assert got["num_corr"] == want["num_corr"] > 15000
    assert frob(got["T"], want["T"]) < 1e-5, frob(got["T"], want["T"])


# ---------------------------------------------------------------------------------------------------------------- scale


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", [600_000, 1_100_000])
def test_scale_beyond_grid_stride_passes(ctx, F, kind, n):
    """132 SMs x 16 blocks x 256 threads = 540 672 queries per grid-stride pass: 600k takes two, 1.1M three."""
    s = synth.textured_sheet_pair(n, seed=n % 97)
    S = Search(ctx, F, kind, s)
    _check_all(S, T0, tag=n)
