"""Dense rigid warp-field ICP on the device (cb_warp_icp_*) at its edges, against the serial oracle in fp32 and fp64
(oracle/warp_field_oracle.cpp) and the float64 normal equations of tests/warp_field_ref.py:
  * sizes at every launch boundary, up to more points than the cooperative CG grid has threads (grid-stride loops);
  * several Gauss-Newton steps on both Huber branches, and the default parameters;
  * general correspondence lists in cb_warp_icp_solve (several pairs per point, duplicates, any order);
  * neighbourhood structure (hub, N[0] != i, n_reg != n, repeated and mutual neighbours, single-entry lists);
  * weights and conditioning, partial overlap, non-finite input and small API edges.

Bars (the device must do as well as the oracle's own arithmetic):
  transforms     |T_dev - T_o64| <= 2 |T_o32 - T_o64| + 8 ulp;
  warped points  |q_dev - q_o32| <= 4 |q_o32 - q_o64| + 16 ulp * side;
  CG solutions   true_rel_residual(delta_dev) <= max(cg_tol, 2 r_o32 + r_o64) on the float64 system of every
                 Gauss-Newton step, each arithmetic at its own iterate;
  counters       gn_steps, converged, cg_iterations equal the fp32 oracle's. Counts that could hinge on the last bits
                 are kept off the edge: cg_tol = 0 with a fixed max_cg_iter, and gn_tol chosen with a margin that the
                 test asserts on the fp64 oracle.
Every case appends a row (worst difference, oracle spread, residuals, bit-equality with the fp32 oracle) to a table
printed at the end of the module (pytest -s)."""
import math

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

import warp_field_ref
from cilantro_b200 import synth

pytestmark = pytest.mark.gpu

ULP = 2.0 ** -24
RES = 0.005
MAX_D2 = 0.04 ** 2
# the reference example's dense weights; cg_tol = 0 and a fixed CG budget keep every count off the last bits
BASE = dict(w_pt=0.1, w_pl=1.0, stiffness=200.0, huber=1e-2, reg_sigma=3 * RES, max_gn_iter=1, gn_tol=0.0,
            max_cg_iter=25, cg_tol=0.0)
REPORT = []


@pytest.fixture(scope="module")
def wf(orc):
    from oracle import warp_field

    return warp_field


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nwarp-field edges: case | max|T_dev-T_o64| | max|T_o32-T_o64| | r_dev | r_o32 | r_o64 | bit-equal to fp32 oracle")
    for row in REPORT:
        print("  " + " | ".join(str(v) for v in row))


def okw(kw):
    """Estimator parameters in the oracle's names."""
    out = {k: v for k, v in kw.items() if k not in ("max_iter", "tol", "max_d2")}
    if "huber" in out:
        out["huber_delta"] = out.pop("huber")
    return out


def identities(n):
    return np.tile(np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32), (n, 1, 1))


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def csr_of_lists(lists, d2_of):
    off = np.concatenate([[0], np.cumsum([len(li) for li in lists])]).astype(np.uint64)
    idx = np.array([v for li in lists for v in li], np.int64)
    val = np.array([d2_of(j, v) for j, li in enumerate(lists) for v in li], np.float32)
    return off, idx, val


def knn_lists(orc, src, k):
    idx, d2, cnt = orc.BruteKnn(src).neighborhoods(src, k, 3.0e38)
    return idx, d2, cnt


class Case:
    """One estimator problem: clouds, the correspondence list and the neighbourhoods. src_w = the source points the
    estimator sees (T_src applied), which is what the oracle takes."""

    def __init__(self, dst, nrm, src, f, s, nb, T_src=None):
        self.dst, self.nrm, self.src, self.f, self.s, self.nb, self.T_src = dst, nrm, src, f, s, nb, T_src

    @property
    def src_w(self):
        from oracle import warp_field

        return self.src if self.T_src is None else warp_field.apply(self.T_src, self.src)

    def device(self, cb, ctx, nb=None):
        dst = cb.Cloud(ctx, self.dst, self.nrm)
        return cb.WarpIcp(ctx, dst, cb.Cloud(ctx, self.src), *(self.nb if nb is None else nb))

    def oracle(self, wf, kw, double):
        return wf.solve(self.dst, self.nrm, self.src_w, self.f, self.s, self.nb, double=double, **okw(kw))

    def system(self, wf, kw, x):
        k = {key: v for key, v in okw(kw).items() if key in ("w_pt", "w_pl", "stiffness", "huber_delta", "reg_sigma")}
        return warp_field_ref.system(wf, self.dst, self.nrm, self.src_w, self.f, self.s, self.nb, x, **k)


def pair_case(orc, n, seed, k=8, **synth_kw):
    P = synth.warp_pair(n, seed=seed, spacing=RES, **synth_kw)
    idx, d2, cnt = knn_lists(orc, P["src"], k)
    from cilantro_b200.capi import neighborhood_csr

    i1, _ = orc.BruteKnn(P["dst"]).query(P["src"], MAX_D2)
    s = np.nonzero(i1 >= 0)[0]
    C = Case(P["dst"], P["dst_normals"], P["src"], i1[s], s, neighborhood_csr(idx, d2, cnt))
    C.P, C.knn = P, (idx, d2, cnt)
    return C


def check_solve(name, cb, ctx, wf, C, kw, icp=None, steps=True, T_mask=None):
    """One cb_warp_icp_solve against both oracles: counters, the transform bar (on T_mask's points if given) and,
    with steps, the residual bar of every Gauss-Newton step. Returns (device result, o32, o64)."""
    icp = icp or C.device(cb, ctx)
    got = icp.solve(C.f, C.s, T_src=C.T_src, **kw)
    o32, o64 = C.oracle(wf, kw, False), C.oracle(wf, kw, True)
    for key in ("gn_steps", "converged", "cg_iterations", "cg_iterations_last"):
        assert got[key] == o32[key], (name, key, got[key], o32[key])
    sel = slice(None) if T_mask is None else T_mask
    Td, T32, T64 = (np.asarray(r["T"], np.float64)[sel] for r in (got, o32, o64))
    err, spread = float(np.abs(Td - T64).max(initial=0)), float(np.abs(T32 - T64).max(initial=0))
    assert err <= 2 * spread + 8 * ULP, (name, err, spread)
    r = [float("nan")] * 3
    if steps:
        r = step_residuals(name, cb, ctx, wf, C, kw, icp, got, o32, o64)
    bit = bool(np.array_equal(bits(got["T"]), bits(o32["T"])) and np.array_equal(bits(got["x"]), bits(o32["x"])))
    REPORT.append((name, f"{err:.3g}", f"{spread:.3g}", *(f"{v:.3g}" for v in r), bit))
    return got, o32, o64


def step_residuals(name, cb, ctx, wf, C, kw, icp, got, o32, o64):
    """The true relative residual, on the float64 system at each arithmetic's own iterate x_{k-1}, of the step
    delta_k = x_k - x_{k-1} it took, for every Gauss-Newton step k. Returns the worst step's (r_dev, r_o32, r_o64)."""
    K = got["gn_steps"]
    prev = [np.zeros((C.src.shape[0], 6))] * 3
    worst = (0.0, 0.0, 0.0)
    for k in range(1, K + 1):
        if k == K:
            cur = [got["x"], o32["x"], o64["x"]]
        else:
            kk = dict(kw, max_gn_iter=k)
            cur = [icp.solve(C.f, C.s, T_src=C.T_src, **kk)["x"], C.oracle(wf, kk, False)["x"],
                   C.oracle(wf, kk, True)["x"]]
        cur = [np.asarray(c, np.float64) for c in cur]
        r = [C.system(wf, kw, p).true_rel_residual(c - p) for c, p in zip(cur, prev)]
        assert r[0] <= max(kw["cg_tol"], 2 * r[1] + r[2]), (name, k, r)
        if r[0] >= worst[0]:
            worst = tuple(r)
        prev = cur
    return worst


def check_points(name, got, o32, o64, src, side):
    from oracle import warp_field

    q = [warp_field.apply(r["T"], src) for r in (got, o32, o64)]
    err, spread = float(np.abs(q[0] - q[1]).max()), float(np.abs(q[1] - q[2]).max())
    assert err <= 4 * spread + 16 * ULP * side, (name, err, spread)
    REPORT.append((name + " (points)", f"{err:.3g}", f"{spread:.3g}", "-", "-", "-",
                   bool(np.array_equal(bits(got["T"]), bits(o32["T"])))))


# ---- 1. sizes at every launch boundary --------------------------------------------------------------------------

def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def device_case(cb, ctx, n, seed, k=8):
    """Correspondences and neighbourhoods from the device searches (bit-exact against brute force in test_gpu_knn)."""
    P = synth.warp_pair(n, seed=seed, spacing=RES)
    dst, src = cb.Cloud(ctx, P["dst"], P["dst_normals"]), cb.Cloud(ctx, P["src"])
    idx, d2, cnt = cb.knn_radius(ctx, src, src, k)
    f, s, _ = cb.find_correspondences(ctx, dst, src, None, MAX_D2)
    C = Case(P["dst"], P["dst_normals"], P["src"], f, s, cb.neighborhood_csr(idx, d2, cnt))
    C.P = P
    return C


@pytest.mark.parametrize("n", [255, 256, 257, 65536, 65537])
def test_sizes_at_block_and_key_width_edges(cb, ctx, wf, n):
    C = device_case(cb, ctx, n, seed=n % 97)
    assert C.s.shape[0] > 0.9 * n
    check_solve(f"n={n}", cb, ctx, wf, C, dict(BASE, max_cg_iter=25))


def test_more_points_than_the_cooperative_grid_has_threads(cb, ctx, wf):
    sm = sm_count()
    upper_bound = 2048 * sm  # resident threads per SM are at most 2048 on sm_90, whatever the occupancy
    n = math.ceil(1.1 * upper_bound)
    assert n > upper_bound
    print(f"\nn = {n}, n / (sm_count x 2048) = {n / upper_bound:.3f} (sm_count {sm})")
    C = device_case(cb, ctx, n, seed=21)
    kw = dict(BASE, max_cg_iter=20)
    icp = C.device(cb, ctx)
    got, o32, _ = check_solve(f"n={n} (grid-stride)", cb, ctx, wf, C, kw, icp=icp)
    est = dict(kw, max_iter=2, tol=0.0, max_d2=MAX_D2)
    e1 = icp.estimate(**est)
    again = icp.solve(C.f, C.s, **kw)
    e2 = icp.estimate(**est)
    fresh = C.device(cb, ctx)
    e_fresh = fresh.estimate(**est)
    s_fresh = fresh.solve(C.f, C.s, **kw)
    for a in (again, s_fresh):  # run to run, after an estimate() on the same object, and on a fresh object
        assert np.array_equal(bits(a["T"]), bits(got["T"])) and np.array_equal(bits(a["x"]), bits(got["x"]))
        assert a["cg_iterations"] == got["cg_iterations"]
    for e in (e2, e_fresh):
        assert np.array_equal(bits(e["T"]), bits(e1["T"]))
        assert (e["iterations"], e["num_corr"], e["cg_iterations"]) == (e1["iterations"], e1["num_corr"],
                                                                        e1["cg_iterations"])
    assert e1["iterations"] == 2 and e1["cg_iterations"] == 2 * 20


# ---- 2. several Gauss-Newton steps --------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def pair2k(orc):
    return pair_case(orc, 2000, seed=3)


@pytest.mark.parametrize("huber", [1e-6, 1e-4, 1e-2, 1e3])
def test_several_gauss_newton_steps(cb, ctx, wf, pair2k, huber):
    C = pair2k
    kw = dict(BASE, huber=huber, max_gn_iter=4, max_cg_iter=30)
    got, _, o64 = check_solve(f"4 GN steps, huber {huber:g}", cb, ctx, wf, C, kw)
    assert got["gn_steps"] == 4 and not got["converged"] and got["cg_iterations"] == 4 * 30
    # which Huber branch the steps after the first use (1e-6: mostly the outer one, 1e3: only the inner one)
    x1 = C.oracle(wf, dict(kw, max_gn_iter=1), True)["x"].astype(np.float64)
    lo, hi = C.system(wf, kw, x1).lo, C.system(wf, kw, x1).hi
    outer = float((np.abs(x1[lo] - x1[hi]) > np.float32(huber)).mean())
    REPORT.append((f"  outer-branch fraction at step 2, huber {huber:g}", f"{outer:.3f}", "", "", "", "", ""))
    if huber == 1e-6:
        assert outer > 0.5
    if huber >= 1e-2:
        assert outer == 0.0
    if huber == 1e-4:
        assert 0.0 < outer < 1.0


def test_gn_tol_stop_with_margin(cb, ctx, wf, pair2k):
    C = pair2k
    kw = dict(BASE, huber=1e-2, max_gn_iter=6, max_cg_iter=30)
    x = [np.zeros((C.src.shape[0], 6))] + [C.oracle(wf, dict(kw, max_gn_iter=k), True)["x"].astype(np.float64)
                                           for k in range(1, 7)]
    d2 = [float(np.max(np.sum((x[k] - x[k - 1]) ** 2, 1))) for k in range(1, 7)]
    # the first step whose max |delta|^2 is at least 4x below the previous one's: gn_tol^2 in between, with a factor
    # of 2 of margin on both sides
    k = next(k for k in range(1, 6) if d2[k] < d2[k - 1] / 4)
    gn_tol = math.sqrt(math.sqrt(d2[k] * d2[k - 1]))
    assert d2[k] < 0.5 * gn_tol ** 2 and d2[k - 1] > 2 * gn_tol ** 2 and all(v > 2 * gn_tol ** 2 for v in d2[:k])
    got, o32, o64 = check_solve(f"gn_tol stop after step {k + 1}", cb, ctx, wf, C, dict(kw, gn_tol=gn_tol))
    assert o64["converged"] and o64["gn_steps"] == k + 1
    assert got["converged"] and got["gn_steps"] == k + 1


def test_default_parameters(cb, ctx, wf, pair2k):
    """cb_warp_default_params (the C++ shim's default): 10 steps, Huber 1e-4, CG to 1e-5."""
    C = pair2k
    p = cb.warp_params()
    kw = dict(w_pt=p.w_pt, w_pl=p.w_pl, stiffness=p.stiffness, huber=p.huber, reg_sigma=1.0,
              max_gn_iter=p.max_gn_iter, gn_tol=p.gn_tol, max_cg_iter=p.max_cg_iter, cg_tol=p.cg_tol)
    assert kw == dict(w_pt=0.0, w_pl=1.0, stiffness=1.0, huber=np.float32(1e-4), reg_sigma=1.0, max_gn_iter=10,
                      gn_tol=np.float32(1e-5), max_cg_iter=1000, cg_tol=np.float32(1e-5))
    assert p.reg_coeff == np.float32(-0.5)
    icp = C.device(cb, ctx)
    got = icp.solve(C.f, C.s)  # the defaults themselves, not the restated ones
    o32, o64 = C.oracle(wf, kw, False), C.oracle(wf, kw, True)
    for key in ("gn_steps", "converged", "cg_iterations", "cg_iterations_last"):
        assert got[key] == o32[key], (key, got[key], o32[key])
    err, spread = np.abs(got["T"] - o64["T"]).max(), np.abs(o32["T"] - o64["T"]).max()
    assert err <= 2 * spread + 8 * ULP, (err, spread)
    # the last step's residual on the float64 system at each arithmetic's own iterate
    K = got["gn_steps"]
    prev = [icp.solve(C.f, C.s, max_gn_iter=K - 1)["x"], C.oracle(wf, dict(kw, max_gn_iter=K - 1), False)["x"],
            C.oracle(wf, dict(kw, max_gn_iter=K - 1), True)["x"]]
    r = [C.system(wf, kw, p_.astype(np.float64)).true_rel_residual(c.astype(np.float64) - p_.astype(np.float64))
         for c, p_ in zip((got["x"], o32["x"], o64["x"]), prev)]
    assert r[0] <= max(kw["cg_tol"], 2 * r[1] + r[2]), r
    REPORT.append((f"defaults, solve ({K} GN steps, {got['cg_iterations']} CG)", f"{err:.3g}", f"{spread:.3g}",
                   *(f"{v:.3g}" for v in r), bool(np.array_equal(bits(got["T"]), bits(o32["T"])))))


def test_default_parameters_through_estimate(cb, ctx, wf, pair2k):
    C = pair2k
    icp = C.device(cb, ctx)
    got = icp.estimate(max_iter=3)  # max_d2 0.01^2, tol 1e-5
    loop = dict(max_iter=3, tol=1e-5, max_d2=1e-4)
    o32 = wf.icp(C.dst, C.nrm, C.src, C.nb, **loop)
    o64 = wf.icp(C.dst, C.nrm, C.src, C.nb, double=True, **loop)
    for key in ("iterations", "converged", "num_corr", "gn_steps", "cg_iterations"):
        assert got[key] == o32[key], (key, got[key], o32[key])
    check_points("defaults, estimate x3", got, o32, o64, C.src, C.P["side"])


# ---- 3. general correspondence lists ------------------------------------------------------------------------------

def multi_pairs(orc, C, seed):
    """1-3 destination points per source point (its nearest ones within MAX_D2, nearest first) and one exact
    duplicate pair, in point order."""
    idx, d2, cnt = orc.BruteKnn(C.dst).neighborhoods(C.src, 3, MAX_D2)
    m = np.minimum(np.random.default_rng(seed).integers(1, 4, C.src.shape[0]), cnt)
    f, s = [], []
    for i in range(C.src.shape[0]):
        for j in range(m[i]):
            f.append(idx[i, j])
            s.append(i)
            if i == 17 and j == 0:  # one exact duplicate
                f.append(idx[i, j])
                s.append(i)
    return np.array(f, np.int64), np.array(s, np.int64)


def shuffle_across_points(s, seed):
    """A permutation of the list that keeps each point's own order."""
    key = np.random.default_rng(seed).permutation(int(s.max()) + 1)[s]
    return np.argsort(key, kind="stable")


def test_general_correspondence_lists(cb, ctx, orc, wf, pair2k):
    C0 = pair2k
    f, s = multi_pairs(orc, C0, seed=1)
    counts = np.bincount(s, minlength=C0.src.shape[0])
    assert counts.max() >= 3 and (counts == 1).any() and (counts == 2).any()
    kw = dict(BASE, max_gn_iter=2, max_cg_iter=30)
    icp = C0.device(cb, ctx)
    results = []
    for seed in (0, 1):
        o = shuffle_across_points(s, seed)
        assert not np.array_equal(o, np.arange(s.shape[0]))
        C = Case(C0.dst, C0.nrm, C0.src, f[o], s[o], C0.nb)
        results.append(check_solve(f"multi-pair list, shuffled ({seed})", cb, ctx, wf, C, kw, icp=icp)[0])
    assert np.array_equal(bits(results[0]["T"]), bits(results[1]["T"]))
    assert np.array_equal(bits(results[0]["x"]), bits(results[1]["x"]))
    # a permutation inside a point changes the fp32 summation order: still within the bars, not necessarily bit-equal
    i3 = np.nonzero(counts == 3)[0][0]
    o = np.arange(s.shape[0])
    sel = np.nonzero(s == i3)[0]
    o[sel] = sel[::-1]
    check_solve("multi-pair list, reversed inside one point", cb, ctx, wf, Case(C0.dst, C0.nrm, C0.src, f[o], s[o],
                                                                                   C0.nb), kw, icp=icp)


def test_large_rotation_of_the_source(cb, ctx, wf, pair2k):
    """T_src = 90 degrees about x plus a translation, the destination moved with it: the estimator sees the same
    problem in a rotated frame."""
    C0 = pair2k
    R = np.array([[1, 0, 0], [0, 0, -1], [0, 1, 0]], np.float32)
    t = np.array([0.1, -0.2, 0.3], np.float32)
    T = np.tile(np.hstack([R, t[:, None]]), (C0.src.shape[0], 1, 1)).astype(np.float32)
    from oracle import warp_field

    dst = warp_field.apply(T[:1].repeat(C0.dst.shape[0], 0), C0.dst)
    nrm = (C0.nrm.astype(np.float64) @ R.T.astype(np.float64)).astype(np.float32)
    C = Case(dst, nrm, C0.src, C0.f, C0.s, C0.nb, T_src=T)
    check_solve("T_src = 90 deg about x", cb, ctx, wf, C, dict(BASE, max_gn_iter=2, max_cg_iter=30))


# ---- 4. neighbourhood structure -----------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def pair1500(orc):
    return pair_case(orc, 1500, seed=7, k=6)


def nbhd_variant(C, variant):
    from cilantro_b200.capi import neighborhood_csr

    idx, d2, cnt = (a.copy() for a in C.knn)
    n = idx.shape[0]
    if variant == "hub":  # every list [i, 0]: point 0 has n - 1 incidences
        return csr_of_lists([[i, 0] for i in range(n)], lambda j, v: float(np.sum((C.src[j] - C.src[v]) ** 2)))
    if variant == "rows shuffled":  # list j belongs to no particular point: N[0] != j
        p = np.random.default_rng(2).permutation(n)
        return neighborhood_csr(idx[p], d2[p], cnt[p])
    if variant == "n_reg < n":
        return neighborhood_csr(idx[: n // 2], d2[: n // 2], cnt[: n // 2])
    if variant == "n_reg > n":
        extra = np.arange(300)[::-1]
        return neighborhood_csr(np.vstack([idx, idx[extra]]), np.vstack([d2, d2[extra]]),
                                np.concatenate([cnt, cnt[extra]]))
    if variant == "repeated neighbour":
        idx[:, 2], d2[:, 2] = idx[:, 1], d2[:, 1]
        return neighborhood_csr(idx, d2, cnt)
    if variant == "single-entry lists":
        cnt[::3] = 1
        return neighborhood_csr(idx, d2, cnt)
    assert variant == "knn"
    return neighborhood_csr(idx, d2, cnt)


@pytest.mark.parametrize("variant", ["knn", "hub", "rows shuffled", "n_reg < n", "n_reg > n", "repeated neighbour",
                                     "single-entry lists"])
def test_neighbourhood_structure(cb, ctx, wf, pair1500, variant):
    C0 = pair1500
    nb = nbhd_variant(C0, variant)
    C = Case(C0.dst, C0.nrm, C0.src, C0.f, C0.s, nb)
    sysd = C.system(wf, BASE, None)
    if variant == "knn":  # mutual neighbours: both (a, b) and (b, a) listed, kept as two arcs
        arcs = sysd.lo * C.src.shape[0] + sysd.hi
        assert arcs.shape[0] - np.unique(arcs).shape[0] > 100
    if variant == "hub":
        assert np.count_nonzero(sysd.lo == 0) == C.src.shape[0] - 1
    if variant == "rows shuffled":
        off, idx, _ = nb
        assert np.count_nonzero(idx[off[:-1].astype(np.int64)] != np.arange(len(off) - 1)) > 0.9 * (len(off) - 1)
    check_solve(f"neighbourhoods: {variant}", cb, ctx, wf, C, dict(BASE, max_gn_iter=2, max_cg_iter=30))


def test_radius_search_csr_equals_the_same_lists_repacked(cb, ctx, wf, pair1500):
    C0 = pair1500
    src = cb.Cloud(ctx, C0.src)
    off, idx, d2 = cb.radius_search(ctx, src, src, (2.5 * RES) ** 2)
    lens = np.diff(off)
    assert lens.min() >= 1 and lens.max() > lens.min() + 3
    # repacked by hand: a padded table (-1 past each length), then its CSR
    tbl_i = np.full((len(lens), lens.max()), -1, np.int64)
    tbl_d = np.zeros(tbl_i.shape, np.float32)
    for j in range(len(lens)):
        tbl_i[j, :lens[j]] = idx[off[j]:off[j + 1]]
        tbl_d[j, :lens[j]] = d2[off[j]:off[j + 1]]
    repacked = cb.neighborhood_csr(tbl_i, tbl_d)
    kw = dict(BASE, max_gn_iter=2, max_cg_iter=30)
    a = C0.device(cb, ctx, (off.astype(np.uint64), idx, d2)).solve(C0.f, C0.s, **kw)
    b = C0.device(cb, ctx, repacked).solve(C0.f, C0.s, **kw)
    assert np.array_equal(bits(a["T"]), bits(b["T"])) and np.array_equal(bits(a["x"]), bits(b["x"]))
    C = Case(C0.dst, C0.nrm, C0.src, C0.f, C0.s, repacked)
    check_solve("neighbourhoods: radius_search CSR", cb, ctx, wf, C, kw)


# ---- 5. weights and conditioning ----------------------------------------------------------------------------------

def test_zero_stiffness(cb, ctx, wf, pair1500):
    C0 = pair1500
    keep = np.random.default_rng(3).random(C0.s.shape[0]) < 0.7
    C = Case(C0.dst, C0.nrm, C0.src, C0.f[keep], C0.s[keep], C0.nb)
    got, o32, _ = check_solve("stiffness 0", cb, ctx, wf, C, dict(BASE, stiffness=0.0, max_gn_iter=2))
    lone = np.setdiff1d(np.arange(C.src.shape[0]), C.s)  # zero diagonal: inv = 1, and the point keeps the identity
    assert lone.shape[0] > 100
    assert np.array_equal(got["T"][lone], identities(lone.shape[0]))
    assert np.array_equal(got["x"][lone], np.zeros((lone.shape[0], 6), np.float32))


def test_rbf_weights_that_underflow(cb, ctx, wf, pair1500):
    C = pair1500
    kw = dict(BASE, reg_sigma=1e-6, max_gn_iter=2)
    assert np.all(C.system(wf, kw, None).c == 0)  # exp(-0.5 d2 / sigma^2) underflows to 0 on every arc
    check_solve("RBF weights underflow to 0", cb, ctx, wf, C, kw)


def test_very_stiff_planar_point_to_plane(cb, ctx, orc, wf):
    P = synth.warp_pair(1500, seed=11, spacing=RES)
    dst = P["dst"].copy()
    dst[:, 2] = 0.0
    nrm = np.tile(np.array([0, 0, 1], np.float32), (dst.shape[0], 1))
    # a common offset (the plane constrains only its z part) plus noise: the in-plane translation and the rotation
    # about z are held only by the arcs, so the system is nearly singular
    offset = np.array([0.003, -0.002, 0.01])
    src = (dst + offset + np.random.default_rng(4).normal(0, 0.002, dst.shape)).astype(np.float32)
    from cilantro_b200.capi import neighborhood_csr

    i1, _ = orc.BruteKnn(dst).query(src, MAX_D2)
    s = np.nonzero(i1 >= 0)[0]
    C = Case(dst, nrm, src, i1[s], s, neighborhood_csr(*knn_lists(orc, src, 6)))
    got, _, _ = check_solve("stiffness 1e6, planar, w_pl only", cb, ctx, wf, C,
                            dict(BASE, w_pt=0.0, w_pl=1.0, stiffness=1e6, max_gn_iter=2))
    assert np.abs(got["T"][:, 2, 3]).max() > 1e-4  # the z offset is being taken out


def test_point_to_point_only_without_normals(cb, ctx, wf, pair1500):
    C0 = pair1500
    C = Case(C0.dst, None, C0.src, C0.f, C0.s, C0.nb)
    check_solve("w_pt only, no normals", cb, ctx, wf, C, dict(BASE, w_pt=1.0, w_pl=0.0, max_gn_iter=2))


def test_point_to_plane_only(cb, ctx, wf, pair1500):
    check_solve("w_pl only", cb, ctx, wf, pair1500, dict(BASE, w_pt=0.0, w_pl=1.0, max_gn_iter=2))


# ---- 6. partial overlap -------------------------------------------------------------------------------------------

def test_partial_overlap(cb, ctx, orc, wf):
    from cilantro_b200.capi import neighborhood_csr

    P = synth.warp_pair(2000, seed=13, spacing=RES)
    src, dst, nrm = P["src"], P["dst"], P["dst_normals"]
    keep = dst[:, 0] < np.quantile(dst[:, 0], 0.7)
    dst, nrm = np.ascontiguousarray(dst[keep]), np.ascontiguousarray(nrm[keep])
    i1, _ = orc.BruteKnn(dst).query(src, (2 * RES) ** 2)
    s = np.nonzero(i1 >= 0)[0]
    n = src.shape[0]
    assert 0.2 < 1 - s.shape[0] / n < 0.45
    # an island far from the cut: its lists stay inside it and no other list reaches it
    idx, d2, cnt = knn_lists(orc, src, 6)
    island = src[:, 0] > np.quantile(src[:, 0], 0.92)
    cut = island[:, None] != island[np.maximum(idx, 0)]
    idx = np.where(cut, -1, idx)
    nb = neighborhood_csr(idx, d2, cnt)
    C = Case(dst, nrm, src, i1[s], s, nb)
    lo_hi = C.system(wf, BASE, None)
    g = sp.coo_matrix((np.ones(lo_hi.lo.shape[0]), (lo_hi.lo, lo_hi.hi)), shape=(n, n))
    _, comp = connected_components(g, directed=False)
    matched = np.zeros(n, bool)
    matched[s] = True
    comp_matched = np.bincount(comp, matched, comp.max() + 1) > 0
    free = ~comp_matched[comp]  # points in arc components without any correspondence
    moved = ~matched & ~free    # unmatched points moved only through arcs
    assert free.sum() > 50 and moved.sum() > 200
    kw = dict(BASE, max_gn_iter=2, max_cg_iter=30)
    got, o32, o64 = check_solve("partial overlap (all points)", cb, ctx, wf, C, kw)
    check_solve("partial overlap (unmatched, moved through arcs)", cb, ctx, wf, C, kw, steps=False, T_mask=moved)
    assert np.abs(got["T"][moved] - identities(int(moved.sum()))).max() > 1e-4
    for r in (got, o32, o64):
        assert np.array_equal(r["T"][free], identities(int(free.sum())))


# ---- 7. non-finite input ------------------------------------------------------------------------------------------

def test_nan_destination_normal(cb, ctx, wf, pair1500):
    """A NaN normal on a matched destination point turns the whole system NaN: the CG runs max_cg_iter iterations
    (|r|^2 < threshold never holds; the device's threshold is FLT_MIN where the oracle's is NaN) and the Gauss-Newton
    loop stops as converged after one step (a NaN |delta|^2 never raises the max). Every transform is NaN."""
    C0 = pair1500
    nrm = C0.nrm.copy()
    nrm[C0.f[10]] = [np.nan, 0.0, 1.0]
    C = Case(C0.dst, nrm, C0.src, C0.f, C0.s, C0.nb)
    kw = dict(BASE, max_gn_iter=3, gn_tol=1e-5, max_cg_iter=20)
    got = C.device(cb, ctx).solve(C.f, C.s, **kw)
    o32, o64 = C.oracle(wf, kw, False), C.oracle(wf, kw, True)
    for o in (o32, o64):
        assert (o["gn_steps"], o["converged"], o["cg_iterations"]) == (1, True, 20)
        assert np.isnan(o["T"]).all() and np.isnan(o["x"]).all() and math.isnan(o["cg_error"])
    assert (got["gn_steps"], got["converged"], got["cg_iterations"], got["cg_iterations_last"]) == (1, True, 20, 20)
    assert np.isnan(got["T"]).all() and np.isnan(got["x"]).all() and math.isnan(got["cg_error"])


def test_inf_source_coordinates(cb, ctx, wf, pair1500):
    """Infinite source points get no correspondence (neither does NaN); with their arcs kept they move with their
    neighbours, like the oracle's."""
    C0 = pair1500
    src = C0.src.copy()
    bad = [5, 77, 300]
    src[5] = np.inf
    src[77] = -np.inf
    src[300] = [np.inf, -np.inf, 0.5]
    icp = cb.WarpIcp(ctx, cb.Cloud(ctx, C0.dst, C0.nrm), cb.Cloud(ctx, src), *C0.nb)
    kw = dict(BASE, max_gn_iter=1, max_cg_iter=30)
    loop = dict(max_iter=3, tol=0.0, max_d2=MAX_D2)
    got = icp.estimate(**kw, **loop)
    f, s, _ = icp.correspondences()
    assert not np.isin(bad, s).any()
    o32 = wf.icp(C0.dst, C0.nrm, src, C0.nb, **loop, **okw(kw))
    o64 = wf.icp(C0.dst, C0.nrm, src, C0.nb, double=True, **loop, **okw(kw))
    for key in ("iterations", "converged", "num_corr", "gn_steps", "cg_iterations"):
        assert got[key] == o32[key], (key, got[key], o32[key])
    assert np.isfinite(got["T"]).all() and np.isfinite(o32["T"]).all()
    err, spread = np.abs(got["T"] - o64["T"]).max(), np.abs(o32["T"] - o64["T"]).max()
    assert err <= 2 * spread + 8 * ULP, (err, spread)
    assert np.abs(got["T"][bad] - identities(3)).max() > 0  # moved through their arcs
    REPORT.append(("Inf source points, estimate x3", f"{err:.3g}", f"{spread:.3g}", "-", "-", "-",
                   bool(np.array_equal(bits(got["T"]), bits(o32["T"])))))


# ---- 8. small API edges -------------------------------------------------------------------------------------------

def test_zero_iterations_returns_t_init(cb, ctx, pair1500):
    C = pair1500
    icp = C.device(cb, ctx)
    icp.estimate(max_iter=1, max_d2=MAX_D2)
    icp.correspondences()  # available after an estimate() with an iteration
    T0 = identities(C.src.shape[0])
    T0[:, :, 3] = np.random.default_rng(5).normal(0, 0.01, (C.src.shape[0], 3)).astype(np.float32)
    got = icp.estimate(T_init=T0, max_iter=0)
    assert got["iterations"] == 0 and not got["converged"] and got["gn_steps"] == 0
    assert np.array_equal(bits(got["T"]), bits(T0))
    with pytest.raises(cb.CbError, match="-1"):
        icp.correspondences()


def test_residuals_without_normals_and_between_estimate_and_correspondences(cb, ctx, wf, pair1500):
    C = pair1500
    T = identities(C.src.shape[0])
    T[:, :, 3] = np.random.default_rng(6).normal(0, 0.003, (C.src.shape[0], 3)).astype(np.float32)
    plain = cb.WarpIcp(ctx, cb.Cloud(ctx, C.dst), cb.Cloud(ctx, C.src), *C.nb)
    got = plain.residuals(T, w_pt=0.7, w_pl=0.0)
    want = wf.residuals(C.dst, None, C.src, T, 0.7, 0.0)
    assert np.array_equal(bits(got), bits(want))
    kw = dict(BASE, max_iter=2, max_d2=MAX_D2)
    a, b = C.device(cb, ctx), C.device(cb, ctx)
    ea, eb = a.estimate(**kw), b.estimate(**kw)
    assert np.array_equal(bits(ea["T"]), bits(eb["T"]))
    la = a.correspondences()
    a.residuals(T, w_pt=0.1, w_pl=1.0)
    b.residuals(T, w_pt=0.1, w_pl=1.0)  # before b's first correspondences() call
    for got_l in (a.correspondences(), b.correspondences()):
        assert all(np.array_equal(x, y) for x, y in zip(got_l, la))
    assert len(la[0]) == ea["num_corr"]
