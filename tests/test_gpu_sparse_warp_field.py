"""Sparse rigid warp-field ICP on the device (cb_sparse_warp_icp_*) against the serial oracle
(oracle/sparse_warp_field_oracle.cpp, fp32 and fp64), scipy and the dense path."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

import cxx
import sparse_warp_field_ref as ref
from cilantro_b200 import synth

pytestmark = pytest.mark.gpu

RES = 0.025  # the reference example's control resolution (examples/non_rigid_icp.cpp:41-43)
RECIPE = dict(w_pt=0.0, w_pl=1.0, stiffness=200.0, huber=1e-2, max_gn_iter=1, gn_tol=5e-4, max_cg_iter=500, cg_tol=1e-5,
              reg_sigma=3.0 * RES, ctrl_sigma=0.5 * RES)
LOOP = dict(max_iter=15, tol=2.5e-3, max_d2=0.02 ** 2)


@pytest.fixture(scope="module")
def swf(orc):
    from oracle import sparse_warp_field

    return sparse_warp_field


@pytest.fixture(scope="module")
def case(orc, cb):
    return ref.make_case(4000, RES, seed=6)


def okw(kw):
    out = dict(kw)
    if "huber" in out:
        out["huber_delta"] = out.pop("huber")
    return out


def make(cb, ctx, P, ctrl=None, m=None, reg=None):
    dst = cb.Cloud(ctx, P["dst"], P["dst_normals"])
    src = cb.Cloud(ctx, P["src"])
    return cb.SparseWarpIcp(ctx, dst, src, P["ctrl"] if ctrl is None else ctrl, P["m"] if m is None else m,
                            P["reg"] if reg is None else reg)


def corr_of(orc, P, max_d2=0.02 ** 2):
    i1, _ = orc.BruteKnn(P["dst"]).query(P["src"], max_d2)
    second = np.nonzero(i1 >= 0)[0]
    return i1[second], second


def true_residual(swf, P, first, second, x, kw):
    """|At At^T x - At b| / |At b| of one step from zero, in fp64 (the oracle's normal equations)."""
    m = P["m"]
    s = swf.system(P["dst"], P["dst_normals"], P["src"], first, second, P["ctrl"], m, P["reg"], np.zeros((m, 6)),
                   np.asarray(x, np.float64), **{k: v for k, v in okw(kw).items() if k in (
                       "w_pt", "w_pl", "stiffness", "huber_delta", "reg_sigma", "ctrl_sigma")})
    return float(np.linalg.norm(s["q"] - s["b"]) / np.linalg.norm(s["b"]))


def test_one_step_against_spsolve(cb, ctx, orc, swf, case):
    P = case
    first, second = corr_of(orc, P)
    m = P["m"]
    kw = dict(RECIPE, max_cg_iter=5000, cg_tol=1e-7)
    At, b = ref.system(P["dst"], P["dst_normals"], P["src"], first, second, P["ctrl"], m, P["reg"], np.zeros((m, 6)),
                       **{k: kw[k] for k in ("w_pt", "w_pl", "stiffness", "huber", "reg_sigma", "ctrl_sigma")})
    AtA = (At @ At.T).tocsc()
    rhs = At @ b
    t = AtA.diagonal() != 0
    want = np.zeros(6 * m)
    want[t] = spla.spsolve(AtA[t][:, t], rhs[t])
    got = make(cb, ctx, P).solve(first, second, **kw)
    res = float(np.linalg.norm(AtA @ got["x"].ravel().astype(np.float64) - rhs) / np.linalg.norm(rhs))
    orc32 = swf.solve(P["dst"], P["dst_normals"], P["src"], first, second, P["ctrl"], m, P["reg"], **okw(kw))
    res32 = float(np.linalg.norm(AtA @ orc32["x"].ravel().astype(np.float64) - rhs) / np.linalg.norm(rhs))
    assert got["gn_steps"] == 1 and got["cg_iterations"] == orc32["cg_iterations"]
    assert res <= 2.0 * res32 + 1e-6, (res, res32)
    assert np.abs(got["x"].ravel() - want).max() < 1e-3 * np.abs(want).max()


def test_loop_matches_the_fp32_oracle(cb, ctx, orc, swf, case):
    P = case
    got = make(cb, ctx, P).estimate(**RECIPE, **LOOP)
    want = swf.icp(P["dst"], P["dst_normals"], P["src"], P["ctrl"], P["m"], P["reg"], **okw(RECIPE), **LOOP)
    assert got["iterations"] == want["iterations"] > 1
    assert got["num_corr"] == want["num_corr"]
    err = np.abs(swf.apply(got["T_dense"], P["src"]) - swf.apply(want["T_dense"], P["src"])).max()
    assert err < 1e-5, err
    assert np.abs(got["T"] - want["T"]).max() < 1e-5
    # the dense field is the resampling of the node transforms
    icp = make(cb, ctx, P)
    np.testing.assert_array_equal(icp.resample(got["T"], ctrl_sigma=RECIPE["ctrl_sigma"]), got["T_dense"])
    np.testing.assert_array_equal(swf.resample(got["T"], P["ctrl"], P["m"], RECIPE["ctrl_sigma"]).view(np.uint32),
                                  got["T_dense"].view(np.uint32))
    # residuals on the dense field: the registration improves the fit
    r = icp.residuals(got["T_dense"], **{k: RECIPE[k] for k in ("w_pt", "w_pl")})
    np.testing.assert_allclose(r, swf.residuals(P["dst"], P["dst_normals"], P["src"], got["T_dense"]), rtol=1e-6,
                               atol=1e-12)
    r0 = icp.residuals(np.tile(np.eye(3, 4, dtype=np.float32), (P["src"].shape[0], 1, 1)))
    assert r.mean() < 0.5 * r0.mean()


def test_one_node_per_point_is_the_dense_path(cb, ctx, orc, case):
    """K = 1 and d2 = 0: every point its own node; the estimator is the dense one."""
    P = synth.warp_pair(1500, seed=9)
    n = P["src"].shape[0]
    idx, d2, cnt = orc.BruteKnn(P["src"]).neighborhoods(P["src"], 12, 3.0e38)
    nb = cb.neighborhood_csr(idx, d2, cnt)
    ctrl = (np.arange(n + 1, dtype=np.uint64), np.arange(n, dtype=np.int64), np.zeros(n, np.float32))
    kw = dict(w_pt=0.1, w_pl=1.0, stiffness=200.0, max_gn_iter=1, gn_tol=5e-4, max_cg_iter=500, cg_tol=1e-5,
              reg_sigma=0.015, max_iter=4, tol=2.5e-3, max_d2=0.04 ** 2, huber=1e-2)
    dst = cb.Cloud(ctx, P["dst"], P["dst_normals"])
    src = cb.Cloud(ctx, P["src"])
    dense = cb.WarpIcp(ctx, dst, src, *nb).estimate(**kw)
    sparse = cb.SparseWarpIcp(ctx, dst, src, ctrl, n, nb).estimate(**kw)
    assert sparse["iterations"] == dense["iterations"] and sparse["cg_iterations"] == dense["cg_iterations"]
    assert np.abs(sparse["T_dense"] - dense["T"]).max() < 1e-5


def test_rigid_motion_is_recovered(cb, ctx, orc):
    from scipy.spatial.transform import Rotation

    P = ref.make_case(3000, RES, seed=8)
    R = Rotation.from_rotvec([0.01, -0.02, 0.015]).as_matrix()
    t = np.array([0.004, -0.003, 0.002])
    P["dst"] = np.ascontiguousarray(P["src"] @ R.T + t, np.float32)
    P["dst_normals"] = np.ascontiguousarray(synth.warp_pair(3000, seed=8)["dst_normals"] @ R.T, np.float32)
    got = make(cb, ctx, P).estimate(**dict(RECIPE, w_pt=1.0, max_gn_iter=5), max_iter=30, tol=1e-6, max_d2=0.02 ** 2)
    warped = np.einsum("nij,nj->ni", got["T_dense"][:, :, :3].astype(np.float64), P["src"]) + got["T_dense"][:, :, 3]
    assert np.abs(warped - P["dst"]).max() < 1e-4


def test_runs_are_bit_identical_and_launches_do_not_depend_on_cg(cb, ctx, case):
    P = case
    icp = make(cb, ctx, P)
    a = icp.estimate(**RECIPE, **LOOP)
    b = icp.estimate(**RECIPE, **LOOP)
    assert a["cg_iterations"] == b["cg_iterations"]
    np.testing.assert_array_equal(a["T"].view(np.uint32), b["T"].view(np.uint32))
    np.testing.assert_array_equal(a["T_dense"].view(np.uint32), b["T_dense"].view(np.uint32))
    few = icp.estimate(**dict(RECIPE, max_cg_iter=3), max_iter=3, tol=0.0, max_d2=LOOP["max_d2"])
    many = icp.estimate(**dict(RECIPE, max_cg_iter=400, cg_tol=1e-9), max_iter=3, tol=0.0, max_d2=LOOP["max_d2"])
    assert few["cg_iterations"] < many["cg_iterations"]
    assert few["kernel_launches"] == many["kernel_launches"]


def test_defined_rules(cb, ctx, orc, swf, case):
    P = case
    n, m = P["src"].shape[0], P["m"]
    off, idx, val = P["ctrl"]
    # rejections
    with pytest.raises(cb.CbError):
        make(cb, ctx, P, ctrl=(off[:-1], idx[:int(off[-2])], val[:int(off[-2])]))  # one list short
    bad = idx.copy()
    bad[5] = m
    with pytest.raises(cb.CbError):
        make(cb, ctx, P, ctrl=(off, bad, val))
    roff, ridx, rval = P["reg"]
    rbad = ridx.copy()
    rbad[3] = m
    with pytest.raises(cb.CbError):
        make(cb, ctx, P, reg=(roff, rbad, rval))
    nonn = cb.Cloud(ctx, P["dst"])
    icpn = cb.SparseWarpIcp(ctx, nonn, cb.Cloud(ctx, P["src"]), P["ctrl"], m, P["reg"])
    with pytest.raises(cb.CbError):
        icpn.estimate(**RECIPE)  # w_pl > 0 without normals
    with pytest.raises(cb.CbError):
        make(cb, ctx, P).estimate(**RECIPE, search_dir="both")
    # duplicates summed, an empty list, an extra node nothing touches: equal to the oracle
    import test_oracle_sparse_warp_field as to

    ctrl = to.with_duplicates(P["ctrl"])
    got = make(cb, ctx, P, ctrl=ctrl, m=m + 1).estimate(**RECIPE, **LOOP)
    want = swf.icp(P["dst"], P["dst_normals"], P["src"], ctrl, m + 1, P["reg"], **okw(RECIPE), **LOOP)
    assert got["iterations"] == want["iterations"]
    assert np.abs(swf.apply(got["T_dense"], P["src"]) - swf.apply(want["T_dense"], P["src"])).max() < 1e-5
    eye = np.eye(3, 4, dtype=np.float32)
    np.testing.assert_array_equal(got["T_dense"][7], eye)  # the empty list
    np.testing.assert_array_equal(got["T"][m], eye)         # the untouched node
    # no data term: identities, the estimator reports false
    s = make(cb, ctx, P).solve(np.zeros(0), np.zeros(0), **RECIPE)
    assert not s["converged"] and s["gn_steps"] == 0
    np.testing.assert_array_equal(s["T"], np.tile(eye, (m, 1, 1)))
    # correspondences after estimate(): the last search's list
    icp = make(cb, ctx, P)
    r = icp.estimate(**RECIPE, max_iter=1, tol=0.0, max_d2=LOOP["max_d2"])
    f, s2, _ = icp.correspondences()
    i1, _ = orc.BruteKnn(P["dst"]).query(P["src"], LOOP["max_d2"])
    assert len(f) == r["num_corr"] and np.array_equal(s2, np.nonzero(i1 >= 0)[0])


def test_large_cloud_step_by_its_fp64_residual(cb, ctx, orc, swf):
    n = int(1.1 * 2048 * ctx.device_info()["sm_count"]) + 1000
    P = ref.make_case(n, RES, seed=10)
    first, second = corr_of(orc, P)
    got = make(cb, ctx, P).solve(first, second, **RECIPE)
    want = swf.solve(P["dst"], P["dst_normals"], P["src"], first, second, P["ctrl"], P["m"], P["reg"], **okw(RECIPE))
    assert got["cg_iterations"] == want["cg_iterations"]
    r_dev = true_residual(swf, P, first, second, got["x"], RECIPE)
    r_orc = true_residual(swf, P, first, second, want["x"], RECIPE)
    assert r_dev <= 2.0 * r_orc + 1e-6, (r_dev, r_orc)


def test_create_destroy_does_not_leak(cb, ctx, case):
    import torch

    P = case
    make(cb, ctx, P).close()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(30):
        icp = make(cb, ctx, P)
        icp.estimate(**RECIPE, max_iter=1, max_d2=LOOP["max_d2"])
        icp.close()
    torch.cuda.synchronize()
    assert free0 - torch.cuda.mem_get_info()[0] < (8 << 20)


def test_cpp_shim_and_example_run(cb, tmp_path):
    import os

    out = cxx.run(cxx.build(os.path.join(cxx.ROOT, "tests", "cpp", "test_sparse_warp_field_shim.cpp"),
                            str(tmp_path / "test_sparse_warp_field_shim")), timeout=600, cwd=str(tmp_path))
    assert "all sparse warp-field shim checks passed" in out
    out = cxx.run(cxx.build(os.path.join(cxx.ROOT, "examples", "sparse_non_rigid_icp_cloud.cpp"),
                            str(tmp_path / "sparse_non_rigid_icp_cloud")), timeout=600, cwd=str(tmp_path))
    line = [ln for ln in out.splitlines() if ln.startswith("mean residual")][0]
    r0, r1 = (float(v) for v in line.split()[2::2])
    assert r1 < 0.5 * r0, line
