"""Sparse control-node warp-field ICP on the device (cb_sparse_warp_icp_*) at its edges, against the serial oracle in
fp32 and fp64 (oracle/sparse_warp_field_oracle.cpp) and the fp64 statement of tests/sparse_warp_field_ref.py:
  * point and node counts at every launch, block and radix-pass boundary, up to more points and nodes than the
    cooperative CG grid has threads (both halves of the matvec stride) and past grid_for's cap in estimate/resample;
  * several Gauss-Newton steps (re-linearised at the blend of the node unknowns) on both Huber branches, the gn_tol
    stop and the default parameters;
  * general correspondence lists in cb_sparse_warp_icp_solve, T_dense_src, T_init and object reuse;
  * control-list structure (ragged, unsorted with duplicates, empty, hub, untouched nodes, m = 1, m = 0, m > n,
    radius-limited lists), control weights that underflow, are subnormal in total or come from +inf distances;
  * resampling of node transforms far apart (both sides of the polar cut-off, reflections, antipodal pairs);
  * non-finite input.

Bars (the device must do as well as the oracle's own arithmetic):
  transforms     |T_dev - T_o64| <= 2 |T_o32 - T_o64| + 8 ulp;
  dense field    |q_dev - q_o32| <= 4 |q_o32 - q_o64| + 16 ulp * side on the warped points;
  CG solutions   |q - b| / |b| of the step on the fp64 normal equations (oracle system() at the step's own iterate)
                 <= max(cg_tol, 2 r_o32 + r_o64), for every Gauss-Newton step;
  counters       gn_steps, converged, cg_iterations and cg_iterations_last equal the fp32 oracle's. cg_tol = 0 with a
                 fixed max_cg_iter, and gn_tol chosen with a margin that the test asserts on the fp64 oracle.
Every case appends a row (worst difference, oracle spread, residuals, bit-equality with the fp32 oracle) to a table
printed at the end of the module (pytest -s)."""
import math

import numpy as np
import pytest

import icp_ref
import sparse_warp_field_ref as ref
from cilantro_b200 import synth

pytestmark = pytest.mark.gpu

ULP = 2.0 ** -24
SP = 0.005       # point spacing of synth.warp_pair
RES = 0.025      # node resolution (the reference example's)
MAX_D2 = 0.02 ** 2
# the reference example's sparse weights plus a point-to-point term; cg_tol = 0 and a fixed CG budget keep every
# count off the last bits
BASE = dict(w_pt=0.1, w_pl=1.0, stiffness=200.0, huber=1e-2, reg_sigma=3 * RES, ctrl_sigma=0.5 * RES, max_gn_iter=1,
            gn_tol=0.0, max_cg_iter=25, cg_tol=0.0)
SYS_KEYS = ("w_pt", "w_pl", "stiffness", "huber_delta", "reg_sigma", "ctrl_sigma")
EMPTY = (np.zeros(1, np.uint64), np.zeros(0, np.int64), np.zeros(0, np.float32))
REPORT = []


@pytest.fixture(scope="module")
def swf(orc):
    from oracle import sparse_warp_field

    return sparse_warp_field


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nsparse warp-field edges: case | max|T_dev-T_o64| | max|T_o32-T_o64| | r_dev | r_o32 | r_o64 | "
          "bit-equal to fp32 oracle")
    for row in REPORT:
        print("  " + " | ".join(str(v) for v in row))


def okw(kw):
    """Estimator parameters in the oracle's names."""
    out = {k: v for k, v in kw.items() if k not in ("max_iter", "tol", "max_d2")}
    if "huber" in out:
        out["huber_delta"] = out.pop("huber")
    return out


def identities(n):
    return np.tile(np.eye(3, 4, dtype=np.float32), (n, 1, 1))


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def csr(lists):
    """(offsets, index, value) of [(nodes, d2s), ...]."""
    off = np.zeros(len(lists) + 1, np.uint64)
    off[1:] = np.cumsum([len(a) for a, _ in lists])
    idx = np.array([v for a, _ in lists for v in a], np.int64)
    val = np.array([v for _, b in lists for v in b], np.float32)
    return off, idx, val


def lists_of(ctrl):
    off, idx, val = (np.asarray(a) for a in ctrl)
    return [(list(idx[off[i]:off[i + 1]]), list(val[off[i]:off[i + 1]])) for i in range(off.shape[0] - 1)]


def arcs_of(reg):
    """The regularisation arcs (lo, hi) of node neighbourhoods in the estimator's rule: (N[0], N[j]), self-arcs
    dropped."""
    off, idx, _ = (np.asarray(a) for a in reg)
    lo, hi = [], []
    for j in range(off.shape[0] - 1):
        nb = idx[int(off[j]):int(off[j + 1])]
        for o in nb[1:]:
            if o != nb[0]:
                lo.append(min(nb[0], o))
                hi.append(max(nb[0], o))
    return np.array(lo, np.int64), np.array(hi, np.int64)


def rel_residual(s):
    nb = float(np.linalg.norm(s["b"]))
    nr = float(np.linalg.norm(s["q"] - s["b"]))
    return nr / nb if nb > 0 else (0.0 if nr == 0 else math.inf)


class Case:
    """One estimator problem: clouds, correspondences (f = dst, s = src index), control lists of the m nodes and the
    node neighbourhoods. T_dense (or None) is the solve's T_dense_src; the oracle takes the warped points."""

    def __init__(self, dst, nrm, src, f, s, ctrl, m, reg, T_dense=None):
        self.dst, self.nrm, self.src, self.f, self.s = dst, nrm, src, f, s
        self.ctrl, self.m, self.reg, self.T_dense = ctrl, int(m), reg, T_dense

    def with_(self, **kw):
        c = Case(self.dst, self.nrm, self.src, self.f, self.s, self.ctrl, self.m, self.reg, self.T_dense)
        for k, v in kw.items():
            setattr(c, k, v)
        return c

    @property
    def src_w(self):
        from oracle import sparse_warp_field

        return self.src if self.T_dense is None else sparse_warp_field.apply(self.T_dense, self.src)

    def device(self, cb, ctx):
        dst = cb.Cloud(ctx, self.dst, self.nrm)
        return cb.SparseWarpIcp(ctx, dst, cb.Cloud(ctx, self.src), self.ctrl, self.m, self.reg)

    def oracle(self, swf, kw, double):
        return swf.solve(self.dst, self.nrm, self.src_w, self.f, self.s, self.ctrl, self.m, self.reg, double=double,
                         **okw(kw))

    def residual(self, swf, kw, x, p):
        k = {key: v for key, v in okw(kw).items() if key in SYS_KEYS}
        return rel_residual(swf.system(self.dst, self.nrm, self.src_w, self.f, self.s, self.ctrl, self.m, self.reg,
                                       x, p, **k))


def corr_brute(orc, dst, src, max_d2=MAX_D2):
    i1, _ = orc.BruteKnn(dst).query(src, max_d2)
    s = np.nonzero(i1 >= 0)[0]
    return i1[s], s


def recipe_case(orc, n, seed, k_ctrl=4):
    """The reference example's recipe (tests/sparse_warp_field_ref.make_case) with brute-force correspondences."""
    P = ref.make_case(n, RES, seed=seed, k_ctrl=k_ctrl, spacing=SP)
    f, s = corr_brute(orc, P["dst"], P["src"])
    C = Case(P["dst"], P["dst_normals"], P["src"], f, s, P["ctrl"], P["m"], P["reg"])
    C.P = P
    return C


def device_case(cb, ctx, n, seed, nodes=None, k_ctrl=4, k_reg=8):
    """Correspondences, control lists and node neighbourhoods from the device searches (bit-exact against brute force
    in test_gpu_knn). nodes: grid_downsample of the source at RES when None."""
    P = synth.warp_pair(n, seed=seed, spacing=SP)
    dst, src = cb.Cloud(ctx, P["dst"], P["dst_normals"]), cb.Cloud(ctx, P["src"])
    if nodes is None:
        nodes = cb.grid_downsample(ctx, P["src"], RES)[0]
    nc = cb.Cloud(ctx, nodes)
    ctrl = cb.neighborhood_csr(*cb.knn_radius(ctx, nc, src, k_ctrl))
    reg = cb.neighborhood_csr(*cb.knn_radius(ctx, nc, nc, min(k_reg, nodes.shape[0])))
    f, s, _ = cb.find_correspondences(ctx, dst, src, None, MAX_D2)
    C = Case(P["dst"], P["dst_normals"], P["src"], f, s, ctrl, nodes.shape[0], reg)
    C.P, C.nodes = P, nodes
    return C


def check_solve(name, cb, ctx, swf, C, kw, icp=None, steps=True, T_mask=None, dev_kw=None):
    """One cb_sparse_warp_icp_solve against both oracles: counters, the transform bar (on T_mask's nodes if given)
    and, with steps, the residual bar of every Gauss-Newton step. The device gets dev_kw when given,
    so that {} runs it on its own defaults; the oracles get kw. Returns (device result, o32, o64)."""
    icp = icp or C.device(cb, ctx)
    dev_kw = kw if dev_kw is None else dev_kw
    got = icp.solve(C.f, C.s, T_dense_src=C.T_dense, **dev_kw)
    o32, o64 = C.oracle(swf, kw, False), C.oracle(swf, kw, True)
    for key in ("gn_steps", "converged", "cg_iterations", "cg_iterations_last"):
        assert got[key] == o32[key], (name, key, got[key], o32[key])
    sel = slice(None) if T_mask is None else T_mask
    Td, T32, T64 = (np.asarray(r["T"], np.float64)[sel] for r in (got, o32, o64))
    err, spread = float(np.abs(Td - T64).max(initial=0)), float(np.abs(T32 - T64).max(initial=0))
    assert err <= 2 * spread + 8 * ULP, (name, err, spread)
    r = [float("nan")] * 3
    if steps:
        r = step_residuals(name, swf, C, kw, icp, got, o32, o64, dev_kw)
    bit = bool(np.array_equal(bits(got["T"]), bits(o32["T"])) and np.array_equal(bits(got["x"]), bits(o32["x"])))
    REPORT.append((name, f"{err:.3g}", f"{spread:.3g}", *(f"{v:.3g}" for v in r), bit))
    return got, o32, o64


def step_residuals(name, swf, C, kw, icp, got, o32, o64, dev_kw):
    """The true relative residual, on the fp64 normal equations at each arithmetic's own iterate x_{k-1}, of the step
    delta_k = x_k - x_{k-1} it took, for every Gauss-Newton step k. Returns the worst step's (r_dev, r_o32, r_o64)."""
    K = got["gn_steps"]
    prev = [np.zeros((C.m, 6))] * 3
    worst = (0.0, 0.0, 0.0)
    for k in range(1, K + 1):
        if k == K:
            cur = [got["x"], o32["x"], o64["x"]]
        else:
            kk = dict(kw, max_gn_iter=k)
            cur = [icp.solve(C.f, C.s, T_dense_src=C.T_dense, **dict(dev_kw, max_gn_iter=k))["x"],
                   C.oracle(swf, kk, False)["x"],
                   C.oracle(swf, kk, True)["x"]]
        cur = [np.asarray(c, np.float64) for c in cur]
        r = [C.residual(swf, kw, p, c - p) for c, p in zip(cur, prev)]
        assert r[0] <= max(kw["cg_tol"], 2 * r[1] + r[2]), (name, k, r)
        if r[0] >= worst[0]:
            worst = tuple(r)
        prev = cur
    return worst


def check_points(name, Td, src, side):
    """The dense-field bar on the warped points; Td = (device, o32, o64) dense transforms."""
    from oracle import sparse_warp_field

    q = [sparse_warp_field.apply(T, src).astype(np.float64) for T in Td]
    err, spread = float(np.abs(q[0] - q[1]).max(initial=0)), float(np.abs(q[1] - q[2]).max(initial=0))
    assert err <= 4 * spread + 16 * ULP * side, (name, err, spread)
    REPORT.append((name + " (points)", f"{err:.3g}", f"{spread:.3g}", "-", "-", "-",
                   bool(np.array_equal(bits(Td[0]), bits(Td[1])))))


def check_transforms(name, T):
    """The transform bar on (device, o32, o64) node transforms."""
    Td, T32, T64 = (np.asarray(t, np.float64) for t in T)
    err, spread = float(np.abs(Td - T64).max(initial=0)), float(np.abs(T32 - T64).max(initial=0))
    assert err <= 2 * spread + 8 * ULP, (name, err, spread)
    REPORT.append((name + " (nodes)", f"{err:.3g}", f"{spread:.3g}", "-", "-", "-",
                   bool(np.array_equal(bits(T[0]), bits(T[1])))))


def check_icp(name, swf, C, got, loop, kw, T_init=None):
    """estimate() against oracle.icp in fp32 (counters) and both arithmetics (node and dense-field bars)."""
    args = (C.dst, C.nrm, C.src, C.ctrl, C.m, C.reg)
    o32 = swf.icp(*args, T_init=T_init, **loop, **okw(kw))
    o64 = swf.icp(*args, T_init=T_init, double=True, **loop, **okw(kw))
    for key in ("iterations", "converged", "num_corr", "gn_steps", "cg_iterations"):
        assert got[key] == o32[key], (name, key, got[key], o32[key])
    check_transforms(name, (got["T"], o32["T"], o64["T"]))
    check_points(name, (got["T_dense"], o32["T_dense"], o64["T_dense"]), C.src, C.P["side"])
    return o32, o64


def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- 1. sizes -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [255, 256, 257, 65536, 65537])
def test_point_counts_at_block_and_grid_edges(cb, ctx, swf, n):
    C = device_case(cb, ctx, n, seed=n % 89)
    assert C.s.shape[0] > 0.9 * n and C.m >= 8
    check_solve(f"n={n}, m={C.m}", cb, ctx, swf, C, dict(BASE, max_gn_iter=2))


@pytest.mark.parametrize("m", [1, 255, 256, 257, 65536, 65537])
def test_node_counts_at_block_and_radix_pass_edges(cb, ctx, swf, m):
    """m source points are the nodes (the radix sort of the node incidence takes 8 key bits up to m = 256, 9 from
    257, 16 up to 65536 and 17 from 65537; sparse_node_kernel's blocks end at multiples of 256)."""
    n = max(4000, m + m // 8)
    P = synth.warp_pair(n, seed=m % 83, spacing=SP)
    nodes = P["src"][np.sort(np.random.default_rng(m).choice(n, m, replace=False))]
    C = device_case(cb, ctx, n, seed=m % 83, nodes=nodes)
    if m == 1:
        assert C.reg[1].shape[0] == 1 and arcs_of(C.reg)[0].shape[0] == 0
    lens = np.diff(C.ctrl[0].astype(np.int64))
    assert lens.min() == min(4, m)
    kw = dict(BASE, max_gn_iter=2)
    if m == 1:  # the one node is up to the cloud's side away: sigma 1 keeps every weight a normal float
        kw["ctrl_sigma"] = 1.0
    check_solve(f"m={m} (n={n})", cb, ctx, swf, C, kw)


def test_more_points_and_nodes_than_the_cooperative_grid_has_threads(cb, ctx, swf):
    """m = n ~ 1.1 x 2048 x sm_count, every point a node with K = 4: both halves of the CG matvec run their grid
    strides, and estimate() and resample() run past grid_for's cap of 8 x sm_count blocks of 256."""
    sm = sm_count()
    upper_bound = 2048 * sm  # resident threads per SM are at most 2048 on sm_90, whatever the occupancy
    n = math.ceil(1.1 * upper_bound)
    assert n > upper_bound and n > 8 * sm * 256
    print(f"\nn = m = {n}, n / (sm_count x 2048) = {n / upper_bound:.3f} (sm_count {sm})")
    P = synth.warp_pair(n, seed=21, spacing=SP)
    C = device_case(cb, ctx, n, seed=21, nodes=P["src"])
    assert C.m == n
    kw = dict(BASE, max_cg_iter=20)
    icp = C.device(cb, ctx)
    got, _, _ = check_solve(f"m = n = {n} (grid-stride)", cb, ctx, swf, C, kw, icp=icp)
    # resample past the cap, bit-identical to the oracle's
    from scipy.spatial.transform import Rotation

    rng = np.random.default_rng(4)
    Tn = np.concatenate([Rotation.from_rotvec(rng.normal(0, 0.3, (n, 3))).as_matrix(),
                         rng.normal(0, 0.01, (n, 3, 1))], 2).astype(np.float32)
    rs = icp.resample(Tn, ctrl_sigma=kw["ctrl_sigma"])
    assert np.array_equal(bits(rs), bits(swf.resample(Tn, C.ctrl, C.m, kw["ctrl_sigma"])))
    REPORT.append((f"m = n = {n}: resample", "-", "-", "-", "-", "-", True))
    # estimate: run to run, after a solve() on the same object, and on a fresh object
    est = dict(kw, max_iter=2, tol=0.0, max_d2=MAX_D2)
    e1 = icp.estimate(**est)
    corr1 = icp.correspondences()  # the search of e1's second iteration
    again = icp.solve(C.f, C.s, **kw)
    e2 = icp.estimate(**est)
    fresh = C.device(cb, ctx)
    e_fresh = fresh.estimate(**est)
    assert np.array_equal(bits(again["T"]), bits(got["T"])) and np.array_equal(bits(again["x"]), bits(got["x"]))
    for e in (e2, e_fresh):
        assert np.array_equal(bits(e["T"]), bits(e1["T"])) and np.array_equal(bits(e["T_dense"]), bits(e1["T_dense"]))
        assert (e["iterations"], e["num_corr"], e["cg_iterations"]) == (e1["iterations"], e1["num_corr"],
                                                                        e1["cg_iterations"])
    assert e1["iterations"] == 2 and e1["cg_iterations"] == 2 * 20
    # e1's last search ran on the points warped by its first iteration's dense field. A fresh one-iteration estimate
    # gives that field: estimate() is bit-identical run to run and across objects, as asserted above
    from oracle import sparse_warp_field

    first = fresh.estimate(**dict(est, max_iter=1))
    warped = sparse_warp_field.apply(first["T_dense"], C.src)
    f, s, _ = cb.find_correspondences(ctx, cb.Cloud(ctx, C.dst, C.nrm), cb.Cloud(ctx, warped), None, MAX_D2)
    o = np.argsort(s, kind="stable")
    assert np.array_equal(corr1[1], s[o]) and np.array_equal(corr1[0], f[o])
    assert len(corr1[0]) == e1["num_corr"]


# ---- 2. several Gauss-Newton steps --------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def case3k(orc):
    return recipe_case(orc, 3000, seed=3)


@pytest.mark.parametrize("huber", [1e-6, 1e-4, 1e-2, 1e3])
def test_several_gauss_newton_steps(cb, ctx, swf, case3k, huber):
    """Steps after the first re-linearise at the blend of the node unknowns and put arcs on the Huber branches."""
    C = case3k
    kw = dict(BASE, huber=huber, max_gn_iter=4, max_cg_iter=30)
    got, _, _ = check_solve(f"4 GN steps, huber {huber:g}", cb, ctx, swf, C, kw)
    assert got["gn_steps"] == 4 and not got["converged"] and got["cg_iterations"] == 4 * 30
    # which Huber branch step 2 uses (1e-6: mostly the outer one, 1e3: only the inner one)
    x1 = C.oracle(swf, dict(kw, max_gn_iter=1), True)["x"].astype(np.float64)
    lo, hi = arcs_of(C.reg)
    outer = float((np.abs(x1[lo] - x1[hi]) > np.float32(huber)).mean())
    REPORT.append((f"  outer-branch fraction at step 2, huber {huber:g}", f"{outer:.3f}", "", "", "", "", ""))
    if huber == 1e-6:
        assert outer > 0.5
    if huber >= 1e-2:
        assert outer == 0.0
    if huber == 1e-4:
        assert 0.0 < outer < 1.0


def test_gn_tol_stop_with_margin(cb, ctx, swf, case3k):
    C = case3k
    kw = dict(BASE, max_gn_iter=6, max_cg_iter=100)
    x = [np.zeros((C.m, 6))] + [C.oracle(swf, dict(kw, max_gn_iter=k), True)["x"].astype(np.float64)
                                for k in range(1, 7)]
    d2 = [float(np.max(np.sum((x[k] - x[k - 1]) ** 2, 1))) for k in range(1, 7)]
    # the first step whose max |delta|^2 is at least 4x below the previous one's: gn_tol^2 in between, with a factor
    # of 2 of margin on both sides
    k = next(k for k in range(1, 6) if d2[k] < d2[k - 1] / 4)
    gn_tol = math.sqrt(math.sqrt(d2[k] * d2[k - 1]))
    assert d2[k] < 0.5 * gn_tol ** 2 and d2[k - 1] > 2 * gn_tol ** 2 and all(v > 2 * gn_tol ** 2 for v in d2[:k])
    got, _, o64 = check_solve(f"gn_tol stop after step {k + 1}", cb, ctx, swf, C, dict(kw, gn_tol=gn_tol))
    assert o64["converged"] and o64["gn_steps"] == k + 1
    assert got["converged"] and got["gn_steps"] == k + 1


def test_default_parameters(cb, ctx, swf, case3k):
    """cb_sparse_warp_default_params (the C++ shim's default): the dense defaults and ctrl_sigma = 1."""
    C = case3k
    p = cb.sparse_warp_params()
    b = p.base
    kw = dict(w_pt=b.w_pt, w_pl=b.w_pl, stiffness=b.stiffness, huber=b.huber, reg_sigma=1.0, ctrl_sigma=1.0,
              max_gn_iter=b.max_gn_iter, gn_tol=b.gn_tol, max_cg_iter=b.max_cg_iter, cg_tol=b.cg_tol)
    assert kw == dict(w_pt=0.0, w_pl=1.0, stiffness=1.0, huber=np.float32(1e-4), reg_sigma=1.0, ctrl_sigma=1.0,
                      max_gn_iter=10, gn_tol=np.float32(1e-5), max_cg_iter=1000, cg_tol=np.float32(1e-5))
    assert b.reg_coeff == np.float32(-0.5) and p.ctrl_coeff == np.float32(-0.5)
    # the device on its defaults themselves (every Gauss-Newton step a call with only max_gn_iter given), the oracles
    # on the restated ones
    got, _, _ = check_solve("defaults, solve", cb, ctx, swf, C, kw, dev_kw={})
    assert got["gn_steps"] > 1


def test_default_parameters_through_estimate(cb, ctx, swf, case3k):
    C = case3k
    got = C.device(cb, ctx).estimate(max_iter=3)  # max_d2 0.01^2, tol 1e-5
    check_icp("defaults, estimate x3", swf, C, got, dict(max_iter=3, tol=1e-5, max_d2=1e-4), {})


# ---- 3. correspondence lists and start states ---------------------------------------------------------------------

def multi_pairs(orc, C, seed):
    """1-3 destination points per source point (its nearest ones within MAX_D2, nearest first) and one exact
    duplicate pair, in point order."""
    idx, _, cnt = orc.BruteKnn(C.dst).neighborhoods(C.src, 3, MAX_D2)
    k = np.minimum(np.random.default_rng(seed).integers(1, 4, C.src.shape[0]), cnt)
    f, s = [], []
    for i in range(C.src.shape[0]):
        for j in range(k[i]):
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


def test_general_correspondence_lists(cb, ctx, orc, swf, case3k):
    C0 = case3k
    f, s = multi_pairs(orc, C0, seed=1)
    counts = np.bincount(s, minlength=C0.src.shape[0])
    assert counts.max() >= 3 and (counts == 1).any() and (counts == 2).any()
    kw = dict(BASE, max_gn_iter=2, max_cg_iter=30)
    icp = C0.device(cb, ctx)
    results = []
    for seed in (0, 1):
        o = shuffle_across_points(s, seed)
        assert not np.array_equal(o, np.arange(s.shape[0]))
        C = C0.with_(f=f[o], s=s[o])
        results.append(check_solve(f"multi-pair list, shuffled ({seed})", cb, ctx, swf, C, kw, icp=icp)[0])
    assert np.array_equal(bits(results[0]["T"]), bits(results[1]["T"]))
    assert np.array_equal(bits(results[0]["x"]), bits(results[1]["x"]))
    # a permutation inside a point changes the fp32 summation order: still within the bars, not necessarily bit-equal
    i3 = np.nonzero(counts == 3)[0][0]
    o = np.arange(s.shape[0])
    sel = np.nonzero(s == i3)[0]
    o[sel] = sel[::-1]
    check_solve("multi-pair list, reversed inside one point", cb, ctx, swf, C0.with_(f=f[o], s=s[o]), kw, icp=icp)


def pivots(src, seed, scale=0.8, offset=2 * SP):
    """Large rotations, different per point, each about a centre c_i = s_i + o_i, o_i ~ N(0, offset^2) per axis:
    T_i s_i = s_i + o_i - R_i o_i moves each point by up to 2 |o_i|, a few point spacings."""
    from scipy.spatial.transform import Rotation

    rng = np.random.default_rng(seed)
    R = Rotation.from_rotvec(rng.normal(0, scale, (src.shape[0], 3))).as_matrix()
    c = src.astype(np.float64) + rng.normal(0, offset, src.shape)
    t = c - np.einsum("nij,nj->ni", R, c)
    return np.concatenate([R, t[:, :, None]], 2).astype(np.float32)


def test_dense_source_transforms(cb, ctx, orc, swf, case3k):
    """The correspondences are those of the warped points. A device that ignored T_dense_src (or read an identity
    field) would solve on the unwarped points: the test shows that this breaks the transform bar."""
    C = case3k.with_(T_dense=pivots(case3k.src, seed=2))
    ang = np.degrees(np.arccos(np.clip((np.trace(C.T_dense[:, :, :3], axis1=1, axis2=2) - 1) / 2, -1, 1)))
    move = np.linalg.norm(C.src_w.astype(np.float64) - C.src, axis=1)
    assert np.median(ang) > 45 and np.median(move) > SP
    f, s = corr_brute(orc, C.dst, C.src_w)
    C = C.with_(f=f, s=s)
    assert s.shape[0] > 0.5 * C.src.shape[0]
    kw = dict(BASE, max_gn_iter=2, max_cg_iter=30)
    _, o32, o64 = check_solve("T_dense_src: per-point rotations", cb, ctx, swf, C, kw)
    ignored = C.with_(T_dense=None).oracle(swf, kw, False)
    err, spread = float(np.abs(ignored["T"] - o64["T"]).max()), float(np.abs(o32["T"] - o64["T"]).max())
    assert err > 10 * (2 * spread + 8 * ULP), (err, spread)
    REPORT.append(("  T_dense_src ignored (fp32 oracle on the unwarped points)", f"{err:.3g}", f"{spread:.3g}", "-",
                   "-", "-", "-"))


def node_init(m, seed):
    from scipy.spatial.transform import Rotation

    rng = np.random.default_rng(seed)
    return np.concatenate([Rotation.from_rotvec(rng.normal(0, 0.01, (m, 3))).as_matrix(),
                           rng.normal(0, 0.002, (m, 3, 1))], 2).astype(np.float32)


def test_estimate_from_t_init_and_object_reuse(cb, ctx, swf, case3k):
    C = case3k
    T0 = node_init(C.m, seed=3)
    kw = dict(BASE, max_cg_iter=30)
    loop = dict(max_iter=3, tol=0.0, max_d2=MAX_D2)
    icp = C.device(cb, ctx)
    got = icp.estimate(T_init=T0, **kw, **loop)
    check_icp("estimate from T_init", swf, C, got, loop, kw, T_init=T0)
    # estimate -> solve(T_dense_src) -> estimate: the solve leaves nothing behind
    icp.solve(C.f, C.s, T_dense_src=pivots(C.src, seed=4), **dict(kw, max_gn_iter=2))
    again = icp.estimate(T_init=T0, **kw, **loop)
    for key in ("T", "T_dense"):
        assert np.array_equal(bits(again[key]), bits(got[key])), key
    assert (again["iterations"], again["num_corr"], again["cg_iterations"]) == (got["iterations"], got["num_corr"],
                                                                                got["cg_iterations"])


# ---- 4. control-list structure ------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def case1500(orc):
    return recipe_case(orc, 1500, seed=7, k_ctrl=12)


def remap_untouched(C):
    """New node numbering with untouched nodes at index 0, as a run of 5 in the middle, and last."""
    m = C.m
    new = np.arange(m) + 1 + 5 * (np.arange(m) >= m // 2)
    off, idx, val = C.ctrl
    roff, ridx, rval = C.reg
    untouched = np.setdiff1d(np.arange(m + 7), new)
    return (off, new[idx], val), m + 7, (roff, new[ridx], rval), untouched


def ctrl_variant(orc, C, variant):
    """(ctrl, m, reg) of a control-list variant of C (12-NN lists of its nodes)."""
    lists = lists_of(C.ctrl)
    n, m, reg = len(lists), C.m, C.reg
    rng = np.random.default_rng(11)
    if variant == "ragged K 1..12":
        ks = rng.integers(1, 13, n)
        lists = [(a[:k], b[:k]) for (a, b), k in zip(lists, ks)]
    elif variant == "unsorted, duplicates":  # reversed, and the nearest node again at the end, 1.5x as far
        lists = [(a[:4][::-1] + a[3:4], b[:4][::-1] + [1.5 * b[3]]) for a, b in lists]
    elif variant == "empty lists interleaved":
        lists = [([], []) if i % 2 else (a[:4], b[:4]) for i, (a, b) in enumerate(lists)]
    elif variant == "hub":  # node 0 last in every list, as heavy as the list's nearest node
        lists = [(a[:4] + [0], b[:4] + b[:1]) for a, b in lists]
    elif variant == "m = 1":  # one node, no arcs: every point blends the same unknowns
        lists = [([0], [0.0]) for _ in lists]
        m, reg = 1, (np.array([0, 1], np.uint64), np.zeros(1, np.int64), np.zeros(1, np.float32))
    elif variant == "m > n":  # the nodes are the source points and 700 more
        extra = C.src[rng.choice(n, 700)] + rng.normal(0, SP, (700, 3)).astype(np.float32)
        nodes = np.concatenate([C.src, extra]).astype(np.float32)
        knn = orc.BruteKnn(nodes)
        from cilantro_b200.capi import neighborhood_csr

        return (neighborhood_csr(*knn.neighborhoods(C.src, 4, 3.0e38)), nodes.shape[0],
                neighborhood_csr(*knn.neighborhoods(nodes, 8, 3.0e38)))
    else:
        assert variant == "K = 4"
        lists = [(a[:4], b[:4]) for a, b in lists]
    return csr(lists), m, reg


@pytest.mark.parametrize("variant", ["K = 4", "ragged K 1..12", "unsorted, duplicates", "empty lists interleaved",
                                     "hub", "m = 1", "m > n"])
def test_control_list_structure(cb, ctx, orc, swf, case1500, variant):
    ctrl, m, reg = ctrl_variant(orc, case1500, variant)
    C = case1500.with_(ctrl=ctrl, m=m, reg=reg)
    lens = np.diff(ctrl[0].astype(np.int64))
    if variant == "ragged K 1..12":
        assert lens.min() == 1 and lens.max() == 12
    if variant == "hub":
        assert all(0 in a for a, _ in lists_of(ctrl))
    if variant == "m > n":
        assert m > C.src.shape[0]
    kw = dict(BASE, max_gn_iter=2, max_cg_iter=30)
    icp = C.device(cb, ctx)
    got, _, _ = check_solve(f"control lists: {variant}", cb, ctx, swf, C, kw, icp=icp)
    Td = icp.resample(got["T"], ctrl_sigma=kw["ctrl_sigma"])
    empty = lens == 0
    assert np.array_equal(Td[empty], identities(int(empty.sum())))
    if variant == "empty lists interleaved":
        assert empty.sum() == C.src.shape[0] // 2


def test_untouched_nodes_first_middle_and_last(cb, ctx, orc, swf, case1500):
    ctrl, m, reg = ctrl_variant(orc, case1500, "K = 4")
    ctrl, m, reg, untouched = remap_untouched(case1500.with_(ctrl=ctrl, m=m, reg=reg))
    assert untouched[0] == 0 and untouched[-1] == m - 1 and untouched.shape[0] == 7
    C = case1500.with_(ctrl=ctrl, m=m, reg=reg)
    got, o32, o64 = check_solve("untouched nodes first, middle, last", cb, ctx, swf, C,
                                dict(BASE, max_gn_iter=2, max_cg_iter=30))
    for r in (got, o32, o64):
        assert np.array_equal(r["T"][untouched], identities(7))
        assert np.array_equal(r["x"][untouched], np.zeros((7, 6), np.float32))


def test_no_nodes(cb, ctx, swf, case1500):
    """n_ctrl = 0: every list empty and no arcs; solve() takes no step and estimate() keeps the identity field."""
    n = case1500.src.shape[0]
    C = case1500.with_(ctrl=(np.zeros(n + 1, np.uint64), np.zeros(0, np.int64), np.zeros(0, np.float32)), m=0,
                       reg=EMPTY)
    kw = dict(BASE, max_gn_iter=2)
    icp = C.device(cb, ctx)
    got = icp.solve(C.f, C.s, **kw)
    o32 = C.oracle(swf, kw, False)
    for key in ("gn_steps", "converged", "cg_iterations", "cg_iterations_last"):
        assert got[key] == o32[key] == 0, (key, got[key], o32[key])
    assert got["T"].shape == (0, 3, 4)
    assert np.array_equal(icp.resample(np.zeros((0, 3, 4), np.float32)), identities(n))
    loop = dict(max_iter=3, tol=1e-5, max_d2=MAX_D2)
    e = icp.estimate(**kw, **loop)
    o = swf.icp(C.dst, C.nrm, C.src, C.ctrl, 0, C.reg, **loop, **okw(kw))
    for key in ("iterations", "converged", "num_corr", "gn_steps", "cg_iterations"):
        assert e[key] == o[key], (key, e[key], o[key])
    assert np.array_equal(e["T_dense"], identities(n)) and np.array_equal(o["T_dense"], identities(n))
    REPORT.append(("n_ctrl = 0", "-", "-", "-", "-", "-", True))


def test_radius_limited_control_lists(cb, ctx, swf, case1500):
    C0 = case1500
    nc, sc = cb.Cloud(ctx, C0.P["nodes"]), cb.Cloud(ctx, C0.src)
    ctrl = cb.neighborhood_csr(*cb.knn_radius(ctx, nc, sc, 4, max_d2=(0.6 * RES) ** 2))
    lens = np.diff(ctrl[0].astype(np.int64))
    assert (lens == 0).sum() > 10 and ((lens > 0) & (lens < 4)).sum() > 100 and (lens == 4).sum() > 10
    C = C0.with_(ctrl=ctrl)
    icp = C.device(cb, ctx)
    kw = dict(BASE, max_gn_iter=2, max_cg_iter=30)
    got, _, _ = check_solve("control lists: knn_radius within 0.6 RES", cb, ctx, swf, C, kw, icp=icp)
    Td = icp.resample(got["T"], ctrl_sigma=kw["ctrl_sigma"])
    assert np.array_equal(Td[lens == 0], identities(int((lens == 0).sum())))


# ---- 5. control weights -------------------------------------------------------------------------------------------

def far_lists(C, every, shift=0.05):
    """Every `every`-th list moved 0.05 further away: with ctrl_sigma = 0.005 its weights exp(-0.5 d2 / sigma^2) are
    below e^-1000 and underflow to 0 in float and double, while the other lists keep weights above e^-40."""
    lists = lists_of(C.ctrl)
    far = np.zeros(len(lists), bool)
    far[::every] = True
    lists = [(a[:4], [v + shift for v in b[:4]] if far[i] else b[:4]) for i, (a, b) in enumerate(lists)]
    return csr(lists), far


def test_some_lists_weights_underflow(cb, ctx, swf, case1500):
    ctrl, far = far_lists(case1500, 3)
    C = case1500.with_(ctrl=ctrl)
    kw = dict(BASE, ctrl_sigma=0.005, max_gn_iter=2, max_cg_iter=30)
    _, _, _, W = ref.sorted_lists(ctrl, kw["ctrl_sigma"])
    assert np.array_equal(W == 0, far) and W[~far].min() > math.exp(-40)
    assert np.isin(np.nonzero(far)[0], C.s).sum() > 200  # matched points with W_i = 0: no data rows, but counted
    icp = C.device(cb, ctx)
    got, _, _ = check_solve("W_i = 0 on every third list", cb, ctx, swf, C, kw, icp=icp)
    Td = icp.resample(got["T"], ctrl_sigma=kw["ctrl_sigma"])
    assert np.array_equal(Td[far], identities(int(far.sum())))


@pytest.mark.parametrize("gn_tol", [0.0, 1e-5])
def test_every_lists_weights_underflow(cb, ctx, swf, case1500, gn_tol):
    """All W_i = 0: b = 0, yet the pairs count, so each Gauss-Newton step runs a CG of no iterations."""
    ctrl, far = far_lists(case1500, 1)
    C = case1500.with_(ctrl=ctrl)
    kw = dict(BASE, ctrl_sigma=0.005, max_gn_iter=3, gn_tol=gn_tol, max_cg_iter=30)
    got = C.device(cb, ctx).solve(C.f, C.s, **kw)
    want = (1, True) if gn_tol > 0 else (3, False)
    for o in (C.oracle(swf, kw, False), C.oracle(swf, kw, True)):
        for key in ("gn_steps", "converged", "cg_iterations", "cg_iterations_last", "cg_error"):
            assert got[key] == o[key], (key, got[key], o[key])
        assert (o["gn_steps"], o["converged"], o["cg_iterations"]) == (*want, 0)
    assert np.array_equal(got["T"], identities(C.m))
    REPORT.append((f"W_i = 0 on every list, gn_tol {gn_tol:g}", "-", "-", "-", "-", "-", True))


def test_subnormal_total_weight(cb, ctx, swf, case1500):
    """A matched point whose one control weight is subnormal in float: 1/W overflows to +inf and its blend is 0 * inf
    = NaN, as in the reference's float arithmetic. The device follows the fp32 oracle: same counters, same NaN
    pattern."""
    lists = [(a[:4], b[:4]) for a, b in lists_of(case1500.ctrl)]
    sigma = 0.005
    i = int(case1500.s[40])
    d2 = np.float32(-2 * sigma ** 2 * math.log(1e-40))  # w = exp(-0.5 d2 / sigma^2) ~ 1e-40
    lists[i] = (lists[i][0][:1], [float(d2)])
    C = case1500.with_(ctrl=csr(lists))
    kw = dict(BASE, ctrl_sigma=sigma, max_gn_iter=2, gn_tol=1e-6, max_cg_iter=20)
    w = np.float32(math.exp(float(np.float32(np.float32(-0.5) / np.float32(sigma * sigma)) * d2)))
    assert 0 < w < np.finfo(np.float32).tiny and np.isinf(np.float32(1) / w)
    got = C.device(cb, ctx).solve(C.f, C.s, **kw)
    o32 = C.oracle(swf, kw, False)
    for key in ("gn_steps", "converged", "cg_iterations", "cg_iterations_last"):
        assert got[key] == o32[key], (key, got[key], o32[key])
    assert np.isnan(o32["x"]).any()
    assert np.array_equal(np.isnan(got["x"]), np.isnan(o32["x"]))
    assert np.array_equal(np.isnan(got["T"]), np.isnan(o32["T"]))
    REPORT.append(("subnormal W_i (fp32: 1/W = inf)", "-", "-", "-", "-", "-",
                   bool(np.array_equal(bits(got["T"]), bits(o32["T"])))))


def test_infinite_control_distance_is_a_zero_weight(cb, ctx, swf, case1500):
    lists = [(a[:4], b[:4]) for a, b in lists_of(case1500.ctrl)]
    for i in range(0, len(lists), 5):
        lists[i] = (lists[i][0], lists[i][1][:2] + [math.inf, math.inf])
    lists[1] = (lists[1][0], [math.inf] * 4)  # all of them: W = 0
    C = case1500.with_(ctrl=csr(lists))
    kw = dict(BASE, max_gn_iter=2, max_cg_iter=30)
    icp = C.device(cb, ctx)
    got, _, _ = check_solve("+inf control distances", cb, ctx, swf, C, kw, icp=icp)
    # the same as dropping those entries
    dropped = csr([([v for v, d in zip(a, b) if d != math.inf], [d for d in b if d != math.inf]) for a, b in lists])
    rd = C.with_(ctrl=dropped).device(cb, ctx).solve(C.f, C.s, **kw)
    assert np.array_equal(bits(rd["T"]), bits(got["T"]))
    Td = icp.resample(got["T"], ctrl_sigma=kw["ctrl_sigma"])
    assert np.array_equal(Td[1], identities(1)[0])


# ---- 6. resampling at its edges -----------------------------------------------------------------------------------

def resample_case(cb, ctx, T, lists):
    """A SparseWarpIcp whose control lists are `lists` over the node transforms T; the clouds do not matter."""
    n = len(lists)
    pts = np.random.default_rng(0).normal(0, 1, (n, 3)).astype(np.float32)
    nrm = np.tile(np.float32([0, 0, 1]), (n, 1))
    C = Case(pts, nrm, pts, np.zeros(0, np.int64), np.zeros(0, np.int64), csr(lists), T.shape[0], EMPTY)
    return C.device(cb, ctx), C.ctrl


def check_resample(name, cb, ctx, swf, T, lists, sigma=1.0, bar=None):
    icp, ctrl = resample_case(cb, ctx, T, lists)
    got = icp.resample(T, ctrl_sigma=sigma)
    o32 = swf.resample(T, ctrl, T.shape[0], sigma)
    st = ref.resample(T, ctrl, sigma)
    R = got[:, :, :3].astype(np.float64)
    assert np.isfinite(got).all()
    assert np.abs(R @ R.transpose(0, 2, 1) - np.eye(3)).max() < 1e-5 and np.abs(np.linalg.det(R) - 1).max() < 1e-5
    sel = slice(None) if bar is None else bar
    err, spread = float(np.abs(got[sel] - st[sel]).max()), float(np.abs(o32[sel] - st[sel]).max())
    assert err <= 2 * spread + 8 * ULP, (name, err, spread)
    REPORT.append((f"resample: {name}", f"{err:.3g}", f"{spread:.3g}", "-", "-", "-",
                   bool(np.array_equal(bits(got), bits(o32)))))
    return got, o32, st


def test_resample_random_rotations(cb, ctx, swf):
    from scipy.spatial.transform import Rotation

    rng = np.random.default_rng(1)
    m, n = 64, 4000
    T = np.concatenate([Rotation.random(m, random_state=2).as_matrix(), rng.normal(0, 1, (m, 3, 1))],
                       2).astype(np.float32)
    lists = [(list(rng.choice(m, k, replace=False)), list(rng.uniform(0, 2, k))) for k in rng.integers(1, 6, n)]
    # the bar where the nearest rotation is well-conditioned (distinct, non-vanishing singular values of the blend);
    # elsewhere only a finite proper rotation
    off, idx, d2 = csr(lists)
    w = ref.rbf(d2, 1.0)
    pt = np.repeat(np.arange(n), np.diff(off).astype(np.int64))
    L = np.zeros((n, 3, 3))
    np.add.at(L, pt, w[:, None, None] * T[idx, :, :3].astype(np.float64))
    sv = np.linalg.svd(L, compute_uv=False)
    ok = (sv[:, 2] > 1e-2 * sv[:, 0]) & (np.abs(np.diff(sv, axis=1)).min(1) > 1e-2 * sv[:, 0])
    assert ok.sum() > 0.5 * n and (np.linalg.det(L[ok]) < 0).sum() > 50
    check_resample("random rotations", cb, ctx, swf, T, lists, bar=ok)


@pytest.mark.parametrize("ratio", [4e-6, 2.5e-7])
def test_resample_at_the_polar_cut_off(cb, ctx, swf, ratio):
    """Even blends of I and Rz(theta), theta near pi, with det(A) / |A|_F^3 = cos^2(theta / 2) just above (polar
    iteration) and below (Jacobi SVD) 1e-6."""
    from scipy.optimize import brentq

    w = np.array([0.5, 0.5])

    def rz(th):
        return np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]])

    th = brentq(lambda t: icp_ref.det_ratio(w[0] * np.eye(3) + w[1] * rz(t)) - ratio, 2.0, np.pi)
    T = np.stack([np.eye(3, 4), np.hstack([rz(th), np.zeros((3, 1))])]).astype(np.float32)
    d2 = [-2 * math.log(v) for v in w]
    lists = [([0, 1], d2)] * 8
    # the float blend the device sees, on the intended side of the cut-off
    wf = np.float32(ref.rbf(np.float32(d2), 1.0))
    A32 = (wf[0] * T[0, :, :3] + wf[1] * T[1, :, :3]) * (np.float32(1) / (wf[0] + wf[1]))
    assert icp_ref.polar_accepts(A32) == (ratio > 1e-6)
    check_resample(f"polar cut-off, det ratio {ratio:g}", cb, ctx, swf, T, lists)


def test_resample_reflection_blends(cb, ctx, swf):
    """Blends with det < 0 and distinct singular values (weights on Rx(pi), Ry(pi), Rz(pi), conjugated by random
    rotations): the reflection is repaired on the largest singular value, LinearTransform::rotation()'s rule."""
    from scipy.spatial.transform import Rotation

    flips = [np.diag([1.0, -1.0, -1.0]), np.diag([-1.0, 1.0, -1.0]), np.diag([-1.0, -1.0, 1.0])]
    Q = Rotation.random(20, random_state=5).as_matrix()
    T = np.concatenate([np.concatenate([Q[k] @ F @ Q[k].T for F in flips]) for k in range(20)]).reshape(60, 3, 3)
    T = np.concatenate([T, np.zeros((60, 3, 1))], 2).astype(np.float32)
    rng = np.random.default_rng(6)
    lists, want = [], []
    for k in range(20):
        while True:  # |a| distinct by 0.05 and det < 0
            w = rng.dirichlet([3, 3, 3])
            a = np.array([w[0] - w[1] - w[2], -w[0] + w[1] - w[2], -w[0] - w[1] + w[2]])  # the blend's diagonal
            s = np.sort(np.abs(a))
            if np.prod(a) < 0 and s[0] > 0.05 and np.diff(s).min() > 0.05:
                break
        lists.append(([3 * k, 3 * k + 1, 3 * k + 2], list(-2 * np.log(w))))
        D = np.sign(a)
        D[np.argmax(np.abs(a))] *= -1  # the largest singular value's direction flipped
        want.append(Q[k] @ np.diag(D) @ Q[k].T)
    got, _, _ = check_resample("reflection blends", cb, ctx, swf, T, lists)
    np.testing.assert_allclose(got[:, :, :3], np.stack(want), atol=1e-5)


def test_resample_antipodal_pairs(cb, ctx, swf):
    """I and a half-turn with equal weights: a rank-deficient blend whose nearest rotation is not unique. Only the
    output's being a finite proper rotation is defined."""
    T = np.stack([np.eye(3, 4), np.diag([-1.0, -1.0, 1.0, 0.0])[:3], np.diag([1.0, -1.0, -1.0, 0.0])[:3]])
    T = T.astype(np.float32)
    lists = [([0, 1], [0.0, 0.0]), ([0, 2], [0.0, 0.0]), ([1, 0], [0.0, 0.0]), ([0, 1, 2], [0.0, 0.0, 0.0])]
    icp, ctrl = resample_case(cb, ctx, T, lists)
    got = icp.resample(T)
    R = got[:, :, :3].astype(np.float64)
    assert np.isfinite(got).all()
    assert np.abs(R @ R.transpose(0, 2, 1) - np.eye(3)).max() < 1e-5 and np.abs(np.linalg.det(R) - 1).max() < 1e-5
    REPORT.append(("resample: antipodal pairs (proper rotation only)", "-", "-", "-", "-", "-",
                   bool(np.array_equal(bits(got), bits(swf.resample(T, ctrl, 3, 1.0))))))


# ---- 7. non-finite input ------------------------------------------------------------------------------------------

def test_nan_destination_normal(cb, ctx, swf, case1500):
    """A NaN normal on a matched destination point turns the whole system NaN: the CG runs max_cg_iter iterations and
    the Gauss-Newton loop stops as converged after one step (a NaN |delta|^2 never raises the max). Every transform
    is NaN."""
    C0 = case1500
    nrm = C0.nrm.copy()
    nrm[C0.f[10]] = [np.nan, 0.0, 1.0]
    C = C0.with_(nrm=nrm)
    kw = dict(BASE, max_gn_iter=3, gn_tol=1e-5, max_cg_iter=20)
    got = C.device(cb, ctx).solve(C.f, C.s, **kw)
    o32, o64 = C.oracle(swf, kw, False), C.oracle(swf, kw, True)
    for o in (o32, o64):
        assert (o["gn_steps"], o["converged"], o["cg_iterations"]) == (1, True, 20)
        assert np.isnan(o["T"]).all() and np.isnan(o["x"]).all() and math.isnan(o["cg_error"])
    assert (got["gn_steps"], got["converged"], got["cg_iterations"], got["cg_iterations_last"]) == (1, True, 20, 20)
    assert np.isnan(got["T"]).all() and np.isnan(got["x"]).all() and math.isnan(got["cg_error"])


def test_inf_source_points(cb, ctx, swf, case1500):
    """Infinite source points get no correspondence; their dense transform is still the blend of their nodes'."""
    C0 = case1500
    ctrl, _, _ = ctrl_variant(None, C0, "K = 4")
    src = C0.src.copy()
    bad = [5, 77, 300]
    src[5] = np.inf
    src[77] = -np.inf
    src[300] = [np.inf, -np.inf, 0.5]
    C = C0.with_(src=src, ctrl=ctrl)
    icp = C.device(cb, ctx)
    kw = dict(BASE, max_cg_iter=30)
    loop = dict(max_iter=3, tol=0.0, max_d2=MAX_D2)
    got = icp.estimate(**kw, **loop)
    _, s, _ = icp.correspondences()
    assert not np.isin(bad, s).any()
    assert np.isfinite(got["T"]).all() and np.isfinite(got["T_dense"]).all()
    assert np.array_equal(bits(got["T_dense"]), bits(icp.resample(got["T"], ctrl_sigma=kw["ctrl_sigma"])))
    assert np.abs(got["T_dense"][bad] - identities(3)).max() > 0
    ok = np.isfinite(src).all(1)
    args = (C.dst, C.nrm, C.src, C.ctrl, C.m, C.reg)
    o32 = swf.icp(*args, **loop, **okw(kw))
    o64 = swf.icp(*args, double=True, **loop, **okw(kw))
    for key in ("iterations", "converged", "num_corr", "gn_steps", "cg_iterations"):
        assert got[key] == o32[key], (key, got[key], o32[key])
    check_transforms("Inf source points, estimate x3", (got["T"], o32["T"], o64["T"]))
    check_points("Inf source points, estimate x3", (got["T_dense"][ok], o32["T_dense"][ok], o64["T_dense"][ok]),
                 src[ok], C0.P["side"])


def test_nan_node_transform_in_t_init(cb, ctx, swf, case1500):
    C0 = case1500
    ctrl, _, _ = ctrl_variant(None, C0, "K = 4")
    C = C0.with_(ctrl=ctrl)
    T0 = node_init(C.m, seed=8)
    T0[3] = np.nan
    kw = dict(BASE, max_cg_iter=30)
    loop = dict(max_iter=2, tol=0.0, max_d2=MAX_D2)
    got = C.device(cb, ctx).estimate(T_init=T0, **kw, **loop)
    args = (C.dst, C.nrm, C.src, C.ctrl, C.m, C.reg)
    o32 = swf.icp(*args, T_init=T0, **loop, **okw(kw))
    for key in ("iterations", "converged", "num_corr", "gn_steps", "cg_iterations"):
        assert got[key] == o32[key], (key, got[key], o32[key])
    for key in ("T", "T_dense"):
        assert np.array_equal(np.isnan(got[key]), np.isnan(o32[key])), key
    nan_pts = np.isnan(o32["T_dense"]).any((1, 2))
    assert nan_pts.sum() > 0 and not nan_pts.all()
    o64 = swf.icp(*args, T_init=T0, double=True, **loop, **okw(kw))
    ok = ~np.isnan(got["T_dense"]).any((1, 2)) & ~np.isnan(o64["T_dense"]).any((1, 2))
    check_points("NaN node in T_init, estimate x2", (got["T_dense"][ok], o32["T_dense"][ok], o64["T_dense"][ok]),
                 C.src[ok], C0.P["side"])
    REPORT.append(("NaN node in T_init: NaN pattern as fp32 oracle", "-", "-", "-", "-", "-",
                   bool(np.array_equal(bits(got["T"]), bits(o32["T"])))))
