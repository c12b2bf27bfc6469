"""Dense rigid warp-field ICP on the device (cb_warp_icp_*) against the serial oracle (oracle/warp_field_oracle.cpp,
in fp32 and fp64) and scipy."""
import os

import numpy as np
import pytest
import scipy.sparse.linalg as spla

import cxx
from cilantro_b200 import synth

ROOT = cxx.ROOT

pytestmark = pytest.mark.gpu

ULP = 2.0 ** -24
# the reference example's dense recipe (examples/non_rigid_icp.cpp), at a 5 mm spacing
RES = 0.005
RECIPE = dict(w_pt=0.1, w_pl=1.0, stiffness=200.0, max_gn_iter=1, gn_tol=5e-4, max_cg_iter=500, cg_tol=1e-5)


@pytest.fixture(scope="module")
def wf(orc):
    from oracle import warp_field

    return warp_field


def nbhd_of(orc, cb, src, k=12):
    idx, d2, cnt = orc.BruteKnn(src).neighborhoods(src, k, 3.0e38)
    return cb.neighborhood_csr(idx, d2, cnt)


def identities(n):
    return np.tile(np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32), (n, 1, 1))


def oracle_kw(kw):
    out = dict(kw)
    if "huber" in out:
        out["huber_delta"] = out.pop("huber")
    return out


@pytest.fixture(scope="module")
def pair(orc, cb):
    P = synth.warp_pair(2000, seed=3, spacing=RES)
    P["nbhd"] = nbhd_of(orc, cb, P["src"])
    return P


def make(cb, ctx, P, nbhd=None, normals=True):
    dst = cb.Cloud(ctx, P["dst"], P["dst_normals"] if normals else None)
    src = cb.Cloud(ctx, P["src"])
    return cb.WarpIcp(ctx, dst, src, *(nbhd if nbhd is not None else P["nbhd"]))


def test_one_gauss_newton_step_against_spsolve(cb, ctx, orc, wf, pair):
    import test_oracle_warp_field as st

    dst, nrm, src = pair["dst"], pair["dst_normals"], pair["src"]
    i1, _ = orc.BruteKnn(dst).query(src, 0.04 ** 2)
    second = np.nonzero(i1 >= 0)[0]
    first = i1[second]
    n = src.shape[0]
    kw = dict(w_pt=0.1, w_pl=1.0, stiffness=200.0, huber=float(np.float32(1e-2)), reg_sigma=3 * RES)
    J, b = st.jacobian(dst, nrm, src, first, second, pair["nbhd"], np.zeros((n, 6)), kw["w_pt"], kw["w_pl"],
                       kw["stiffness"], kw["huber"], kw["reg_sigma"])
    delta = spla.spsolve((J.T @ J).tocsc(), J.T @ b).reshape(n, 6)
    want = np.stack([np.hstack([st.drot(*d[:3])[0], d[3:, None]]) for d in delta])
    icp = make(cb, ctx, pair)
    prm = dict(kw, max_gn_iter=1, max_cg_iter=5000, cg_tol=1e-5)
    got = icp.solve(first, second, **prm)
    again = icp.solve(first, second, **prm)
    assert np.array_equal(got["T"].view(np.uint32), again["T"].view(np.uint32)), "not bit-identical run to run"
    assert got["cg_error"] <= 1e-5 and got["gn_steps"] == 1 and got["cg_iterations"] > 0
    o32 = wf.solve(dst, nrm, src, first, second, pair["nbhd"], **oracle_kw(prm))
    o64 = wf.solve(dst, nrm, src, first, second, pair["nbhd"], double=True, **oracle_kw(prm))
    # the true relative residual |A x - b| / |b| on the float64 system. A float solution vector cannot go below the
    # residual of the float64 CG solution rounded to float (the system is stiff: that floor is above cg_tol here), and
    # the fp32 recurrence of CG (the reference's arithmetic, restated by the fp32 oracle) drifts from the true residual
    # while its own recursive residual reaches cg_tol (asserted above). The device must do as well as that arithmetic.
    A, g = (J.T @ J).tocsr(), J.T @ b
    rel = lambda x: float(np.linalg.norm(A @ x.astype(np.float64).reshape(-1) - g) / np.linalg.norm(g))  # noqa: E731
    r_dev, r_o32, r_floor = rel(got["x"]), rel(o32["x"]), rel(o64["x"])
    assert o64["cg_error"] <= 1e-5
    assert r_dev <= max(1e-5, 2 * r_o32 + r_floor), (r_dev, r_o32, r_floor)
    err_dev = np.abs(got["T"] - want).max()
    err_o32 = np.abs(o32["T"] - want).max()
    # floor: both solutions are stored as float transforms, so either error can sit at a few ulps of the largest
    # entry (the rotation's ~1) even when the CG is exact; 8 ulps covers the conversion of the angles as well
    assert err_dev <= 2 * err_o32 + 8 * ULP, (err_dev, err_o32)


def test_whole_icp_against_oracle(cb, ctx, orc, wf, pair):
    dst, nrm, src = pair["dst"], pair["dst_normals"], pair["src"]
    kw = dict(RECIPE, huber=1e-2, reg_sigma=3 * RES)
    loop = dict(max_iter=15, tol=2.5e-3, max_d2=0.04 ** 2)
    icp = make(cb, ctx, pair)
    got = icp.estimate(**kw, **loop)
    o32 = wf.icp(dst, nrm, src, pair["nbhd"], **loop, **oracle_kw(kw))
    o64 = wf.icp(dst, nrm, src, pair["nbhd"], double=True, **loop, **oracle_kw(kw))
    assert got["iterations"] == o32["iterations"]
    assert got["converged"] == o32["converged"]
    # tolerances from the spread of the two oracle arithmetics
    q_dev, q32, q64 = (wf.apply(T, src) for T in (got["T"], o32["T"], o64["T"]))
    spread = np.abs(q32 - q64).max()
    assert np.abs(q_dev - q32).max() <= 4 * spread + 16 * ULP * pair["side"], (np.abs(q_dev - q32).max(), spread)
    assert abs(got["num_corr"] - o32["num_corr"]) <= max(2 * abs(o32["num_corr"] - o64["num_corr"]), 2)
    r0 = wf.residuals(dst, nrm, src, identities(src.shape[0]), 0.1, 1.0).mean()
    r1 = icp.residuals(got["T"], **kw).mean()
    assert r1 < 0.5 * r0, (r1, r0)
    # residuals of given transforms: bit for bit; correspondences: those of cb_find_correspondences on the warped points
    want_r = wf.residuals(dst, nrm, src, got["T"], 0.1, 1.0)
    assert np.array_equal(icp.residuals(got["T"], **kw).view(np.uint32), want_r.view(np.uint32))
    T_prev = got["T"]  # the last search ran on the transforms before the last update: search once more from these
    one = icp.estimate(T_init=T_prev, **dict(kw, max_iter=1, tol=0.0, max_d2=0.04 ** 2))
    f, s, v = icp.correspondences()
    warped = cb.Cloud(ctx, wf.apply(T_prev, src))
    ef, es, ev = cb.find_correspondences(ctx, icp.dst, warped, None, 0.04 ** 2)
    assert np.array_equal(f, ef) and np.array_equal(s, es) and np.array_equal(v.view(np.uint32), ev.view(np.uint32))
    assert one["num_corr"] == len(f)


def test_rigid_motion_is_recovered(cb, ctx, orc):
    P = synth.warp_pair(1500, seed=5, spacing=RES, bend=0.0, noise=0.0)
    dst = P["dst"].astype(np.float64)
    th = np.deg2rad(2.0)
    R = np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]])
    t = np.array([0.004, -0.002, 0.003])
    c = dst.mean(0)
    src = ((dst - c) @ R.T + c + t).astype(np.float32)
    P["src"] = src
    nb = nbhd_of(orc, cb, src)
    icp = make(cb, ctx, P, nb)
    got = icp.estimate(w_pt=1.0, w_pl=1.0, stiffness=1e4, huber=1e-2, reg_sigma=3 * RES, max_iter=30, tol=1e-5,
                       max_d2=0.02 ** 2, max_gn_iter=1, max_cg_iter=1000)
    Tinv = np.hstack([R.T, (c - R.T @ (c + t))[:, None]])  # dst = R^T (src - c - t) + c
    err = np.linalg.norm((got["T"].astype(np.float64) - Tinv[None]).reshape(-1, 12), axis=1).max()
    assert got["converged"], got
    assert err < 1e-3, err


def test_launch_count_does_not_depend_on_cg_iterations(cb, ctx, pair):
    icp = make(cb, ctx, pair)
    kw = dict(RECIPE, max_iter=1, cg_tol=0.0, max_gn_iter=1, reg_sigma=3 * RES, max_d2=0.04 ** 2)
    a = icp.estimate(**dict(kw, max_cg_iter=10))
    b = icp.estimate(**dict(kw, max_cg_iter=500))
    assert a["cg_iterations"] == 10 and b["cg_iterations"] == 500
    assert a["kernel_launches"] == b["kernel_launches"]


def test_small_and_degenerate_inputs(cb, ctx, orc, wf):
    for n in (0, 1, 2):
        P = synth.warp_pair(max(n, 1), seed=n)
        P["src"] = P["src"][:n]
        nb = (np.arange(n + 1, dtype=np.uint64) * min(n, 2), np.zeros(0, np.int64), np.zeros(0, np.float32))
        if n:
            i, d2, c = orc.BruteKnn(P["src"]).neighborhoods(P["src"], 2, 3.0e38)
            nb = cb.neighborhood_csr(i, d2, c)
        icp = make(cb, ctx, P, nb)
        got = icp.estimate(max_d2=1.0)
        assert got["T"].shape == (n, 3, 4)
        want = wf.icp(P["dst"], P["dst_normals"], P["src"], nb, max_d2=1.0)
        assert got["iterations"] == want["iterations"]
        assert np.abs(got["T"] - want["T"]).max() < 1e-4 if n else True


def test_neighbourhood_rules_and_rejections(cb, ctx, orc, wf, pair):
    n = pair["src"].shape[0]
    empty = (np.zeros(n + 1, np.uint64), np.zeros(0, np.int64), np.zeros(0, np.float32))
    selfs = (np.arange(n + 1, dtype=np.uint64) * 2, np.repeat(np.arange(n), 2), np.zeros(2 * n, np.float32))
    kw = dict(max_iter=2, max_d2=0.04 ** 2)
    a = make(cb, ctx, pair, empty).estimate(**kw)
    b = make(cb, ctx, pair, selfs).estimate(**kw)
    assert np.array_equal(a["T"].view(np.uint32), b["T"].view(np.uint32))
    bad = (np.array([0, 2], np.uint64), np.array([0, n], np.int64), np.zeros(2, np.float32))
    with pytest.raises(cb.CbError, match="-1"):
        make(cb, ctx, pair, bad)
    icp = make(cb, ctx, pair, normals=False)
    with pytest.raises(cb.CbError, match="-1"):
        icp.estimate(w_pl=1.0)
    got = icp.estimate(w_pt=1.0, w_pl=0.0, max_iter=1, max_d2=0.04 ** 2)  # point-to-point only needs no normals
    assert got["num_corr"] > 0
    icp = make(cb, ctx, pair)
    for opt in (dict(search_dir="both"), dict(require_reciprocal=True), dict(one_to_one=True),
                dict(inlier_fraction=0.5)):
        with pytest.raises(cb.CbError, match="-5"):
            icp.estimate(**opt)
    sharded = cb.Cloud(ctx, pair["src"], index_offset=10)
    with pytest.raises(cb.CbError, match="-5"):
        cb.WarpIcp(ctx, icp.dst, sharded, *pair["nbhd"])


def test_non_finite_points_and_zero_cg_iterations(cb, ctx, orc, wf, pair):
    P = dict(pair)
    src = pair["src"].copy()
    src[[5, 77]] = np.nan
    P["src"] = src
    # point 5 keeps its arcs; point 77 has none
    off, idx, val = pair["nbhd"]
    lists = []
    for j in range(len(off) - 1):
        li, lv = idx[off[j]:off[j + 1]], val[off[j]:off[j + 1]]
        lists.append((li[:0], lv[:0]) if j == 77 else (li[li != 77], lv[li != 77]))
    nb = (np.concatenate([[0], np.cumsum([len(li) for li, _ in lists])]).astype(np.uint64),
          np.concatenate([li for li, _ in lists]), np.concatenate([lv for _, lv in lists]))
    icp = make(cb, ctx, P, nb)
    got = icp.estimate(max_iter=3, max_d2=0.04 ** 2, **dict(RECIPE, reg_sigma=3 * RES))
    f, s, v = icp.correspondences()
    assert 5 not in s and 77 not in s
    assert np.array_equal(got["T"][77], identities(1)[0])
    assert np.isfinite(got["T"]).all()
    z = icp.estimate(max_iter=2, max_d2=0.04 ** 2, **dict(RECIPE, max_cg_iter=0))
    assert z["cg_iterations"] == 0 and np.array_equal(z["T"], identities(src.shape[0]))


def test_cpp_shim_runs(cb, tmp_path):
    out = cxx.run(cxx.build(os.path.join(ROOT, "tests", "cpp", "test_warp_field_shim.cpp"),
                            str(tmp_path / "test_warp_field_shim")), timeout=600, cwd=str(tmp_path))
    assert "all warp-field shim checks passed" in out


def test_example_program_registers_the_synthetic_pair(cb, tmp_path):
    out = cxx.run(cxx.build(os.path.join(ROOT, "examples", "non_rigid_icp_cloud.cpp"),
                            str(tmp_path / "non_rigid_icp_cloud")), timeout=600, cwd=str(tmp_path))
    line = [ln for ln in out.splitlines() if ln.startswith("mean residual")][0]
    r0, r1 = (float(v) for v in line.split()[2::2])
    assert r1 < 0.5 * r0, line
