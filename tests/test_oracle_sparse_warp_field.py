"""The sparse warp-field oracle (oracle/sparse_warp_field_oracle.cpp) against a scipy statement of the reference's
linear system (tests/sparse_warp_field_ref.py), and that statement against finite differences. No GPU."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

import sparse_warp_field_ref as ref

KW = dict(w_pt=0.1, w_pl=1.0, stiffness=200.0, huber=1e-2, reg_sigma=0.075, ctrl_sigma=0.0125)


@pytest.fixture(scope="module")
def swf():
    from oracle import sparse_warp_field

    sparse_warp_field.build()
    return sparse_warp_field


@pytest.fixture(scope="module")
def case():
    return ref.make_case(600, 0.025, seed=4)


def corr_of(P, max_d2=0.02 ** 2):
    import oracle

    i1, _ = oracle.BruteKnn(P["dst"]).query(P["src"], max_d2)
    second = np.nonzero(i1 >= 0)[0]
    return i1[second], second


def with_duplicates(ctrl):
    """Every fifth list gets its first node again (duplicates are summed) and list 7 is emptied (identity)."""
    off, idx, val = (np.asarray(a) for a in ctrl)
    lists = [(list(idx[off[i]:off[i + 1]]), list(val[off[i]:off[i + 1]])) for i in range(off.shape[0] - 1)]
    for i in range(0, len(lists), 5):
        lists[i][0].append(lists[i][0][0])
        lists[i][1].append(lists[i][1][0] * 1.5)
    lists[7] = ([], [])
    o = np.zeros(len(lists) + 1, np.uint64)
    o[1:] = np.cumsum([len(a) for a, _ in lists])
    return o, np.array(sum((a for a, _ in lists), []), np.int64), np.array(sum((b for _, b in lists), []), np.float32)


def oracle_kw(kw):
    out = dict(kw)
    out["huber_delta"] = out.pop("huber")
    return out


def test_reference_statement_is_the_jacobian_of_its_residuals(case):
    """At^T = d(model)/dX by central differences: the data rows are the chain rule through the blended unknowns and
    the regularisation rows the Huber derivative; b = the residuals."""
    P = dict(case)
    P["src"] = P["src"][:60]
    off, idx, val = P["ctrl"]
    P["ctrl"] = (off[:61], idx[:int(off[60])], val[:int(off[60])])
    first, second = corr_of(P, 0.03 ** 2)
    m = P["m"]
    rng = np.random.default_rng(2)
    x = rng.normal(0, 0.02, (m, 6))
    kw = dict(KW)
    args = (P["dst"], P["dst_normals"], P["src"], first, second, P["ctrl"], m, P["reg"])
    At, b = ref.system(*args, x, **kw)

    def model(xv):  # J x = b with J = d(model)/dx: model = -(residual) up to the constant destination terms
        _, bb = ref.system(*args, xv.reshape(m, 6), **kw)
        return -bb

    eps = 1e-6
    cols = rng.choice(6 * m, 25, replace=False)
    J = At.T.toarray()
    for c in cols:
        e = np.zeros(6 * m)
        e[c] = eps
        fd = (model(x.ravel() + e) - model(x.ravel() - e)) / (2 * eps)
        np.testing.assert_allclose(J[:, c], fd, rtol=1e-5, atol=1e-7)
    assert b.shape[0] == At.shape[1]


def test_resample_statement_blends_and_projects():
    rng = np.random.default_rng(0)
    from scipy.spatial.transform import Rotation

    T = np.concatenate([Rotation.random(5, random_state=1).as_matrix(), rng.normal(0, 1, (5, 3, 1))], 2)
    ctrl = (np.array([0, 1, 3, 3]), np.array([2, 0, 4]), np.array([0.0, 0.1, 0.4], np.float32))
    out = ref.resample(T, ctrl, 0.5)
    np.testing.assert_allclose(out[0], T[2], atol=1e-12)
    np.testing.assert_allclose(out[2], np.hstack([np.eye(3), np.zeros((3, 1))]), atol=0)
    w = ref.rbf(np.float32([0.1, 0.4]), 0.5)
    blend = (w[0] * T[0] + w[1] * T[4]) / w.sum()
    np.testing.assert_allclose(out[1, :, 3], blend[:, 3], atol=1e-12)
    assert abs(np.linalg.det(out[1, :, :3]) - 1) < 1e-12
    U, _, Vt = np.linalg.svd(blend[:, :3])
    np.testing.assert_allclose(out[1, :, :3], U @ Vt, atol=1e-12)


@pytest.mark.parametrize("dups", [False, True])
def test_oracle_normal_equations_match_the_reference_layout(swf, case, dups):
    P = dict(case)
    if dups:
        P["ctrl"] = with_duplicates(P["ctrl"])
    first, second = corr_of(P)
    m = P["m"]
    rng = np.random.default_rng(5)
    x = rng.normal(0, 0.01, (m, 6))
    p = rng.normal(0, 1, (m, 6))
    At, b = ref.system(P["dst"], P["dst_normals"], P["src"], first, second, P["ctrl"], m, P["reg"], x, **KW)
    got = swf.system(P["dst"], P["dst_normals"], P["src"], first, second, P["ctrl"], m, P["reg"], x, p,
                     **oracle_kw(KW))
    AtA = (At @ At.T).tocsr()
    np.testing.assert_allclose(got["b"].ravel(), At @ b, rtol=1e-9, atol=1e-12 * np.abs(At @ b).max())
    np.testing.assert_allclose(got["diag"].ravel(), AtA.diagonal(), rtol=1e-9, atol=1e-12 * AtA.diagonal().max())
    q = AtA @ p.ravel()
    np.testing.assert_allclose(got["q"].ravel(), q, rtol=1e-9, atol=1e-11 * np.abs(q).max())


def test_oracle_fp64_step_matches_spsolve(swf, case):
    P = case
    first, second = corr_of(P)
    m = P["m"]
    At, b = ref.system(P["dst"], P["dst_normals"], P["src"], first, second, P["ctrl"], m, P["reg"], np.zeros((m, 6)),
                       **KW)
    AtA = (At @ At.T).tocsc()
    rhs = At @ b
    touched = AtA.diagonal() != 0  # nodes no point and no arc touches keep x = 0
    want = np.zeros(6 * m)
    want[touched] = spla.spsolve(AtA[touched][:, touched], rhs[touched])
    got = swf.solve(P["dst"], P["dst_normals"], P["src"], first, second, P["ctrl"], m, P["reg"], max_gn_iter=1,
                    max_cg_iter=100000, cg_tol=1e-14, double=True, **oracle_kw(KW))
    assert got["gn_steps"] == 1
    np.testing.assert_allclose(got["x"].ravel(), want, atol=2e-6 * np.abs(want).max())


def test_oracle_resample_matches_the_statement(swf, case):
    from scipy.spatial.transform import Rotation

    P = case
    m = P["m"]
    rng = np.random.default_rng(3)
    T = np.concatenate([Rotation.from_rotvec(rng.normal(0, 0.05, (m, 3))).as_matrix(),
                        rng.normal(0, 0.01, (m, 3, 1))], 2).astype(np.float32)
    ctrl = with_duplicates(P["ctrl"])
    got = swf.resample(T, ctrl, m, KW["ctrl_sigma"])
    want = ref.resample(T, ctrl, KW["ctrl_sigma"])
    np.testing.assert_allclose(got, want, atol=2e-6)
    np.testing.assert_array_equal(got[7], np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32))


def test_oracle_fp32_loop_tracks_fp64(swf, case):
    P = case
    kw = dict(oracle_kw(KW), max_gn_iter=1, gn_tol=5e-4, max_cg_iter=500, cg_tol=1e-5)
    a = swf.icp(P["dst"], P["dst_normals"], P["src"], P["ctrl"], P["m"], P["reg"], max_iter=4, tol=2.5e-3,
                max_d2=0.02 ** 2, **kw)
    b = swf.icp(P["dst"], P["dst_normals"], P["src"], P["ctrl"], P["m"], P["reg"], max_iter=4, tol=2.5e-3,
                max_d2=0.02 ** 2, double=True, **kw)
    assert a["iterations"] == b["iterations"] > 0
    wa = swf.apply(a["T_dense"], P["src"])
    wb = swf.apply(b["T_dense"], P["src"])
    assert np.abs(wa - wb).max() < 1e-4
    # the registration improves the fit: mean point-to-plane residual drops
    r0 = swf.residuals(P["dst"], P["dst_normals"], P["src"], np.tile(np.eye(3, 4, dtype=np.float32), (len(wa), 1, 1)))
    r1 = swf.residuals(P["dst"], P["dst_normals"], P["src"], a["T_dense"])
    assert r1.mean() < r0.mean()
