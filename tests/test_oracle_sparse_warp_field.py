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


def test_resample_repairs_a_reflection_blend_on_the_largest_singular_value(swf):
    """A blend of rotations far apart can have det < 0: weights (0, .45, .33, .22) on I, Rx(pi), Ry(pi), Rz(pi) give
    diag(-.10, -.34, -.56). LinearTransform::rotation() (space_transformations.hpp:43-51) negates column 0 of U, the
    largest singular value's (Eigen's JacobiSVD sorts them descending): the result is diag(-1, -1, 1) = Rz(pi), where
    the Kabsch rule (column 2, the smallest) would give Rx(pi). Also conjugated by a random rotation Q, which keeps the
    singular values and moves the answer to Q Rz(pi) Q^T."""
    from scipy.spatial.transform import Rotation

    rots = [np.eye(3), np.diag([1.0, -1.0, -1.0]), np.diag([-1.0, 1.0, -1.0]), np.diag([-1.0, -1.0, 1.0])]
    w = np.array([0.45, 0.33, 0.22])
    sigma = 1.0
    # d2 = +inf is a zero weight; the others reproduce w up to a common factor
    d2 = np.concatenate([[np.inf], -2.0 * sigma ** 2 * np.log(w)]).astype(np.float32)
    t = np.array([[0.1, 0.2, 0.3], [-1.0, 0.5, 2.0], [0.3, -0.7, 0.0], [2.0, 1.0, -1.0]])
    Q = Rotation.random(random_state=7).as_matrix()
    ctrl = (np.array([0, 4, 8], np.uint64), np.array([0, 1, 2, 3, 4, 5, 6, 7], np.int64), np.concatenate([d2, d2]))
    T = np.concatenate([np.concatenate([np.stack(rots), t[:, :, None]], 2),
                        np.concatenate([Q @ np.stack(rots) @ Q.T, t[:, :, None]], 2)]).astype(np.float32)
    A = np.einsum("k,kij->ij", ref.rbf(d2, sigma), T[:4, :, :3].astype(np.float64)) / ref.rbf(d2, sigma).sum()
    np.testing.assert_allclose(A, np.diag([-0.10, -0.34, -0.56]), atol=1e-6)
    assert np.linalg.det(A) < 0
    want_R = [np.diag([-1.0, -1.0, 1.0]), Q @ np.diag([-1.0, -1.0, 1.0]) @ Q.T]  # sign(A) with the largest's flipped
    w_all = ref.rbf(d2, sigma)
    want_t = (w_all[:, None] * t).sum(0) / w_all.sum()
    helper = ref.resample(T, ctrl, sigma)
    orc = swf.resample(T, ctrl, 8, sigma)
    for i in range(2):
        np.testing.assert_allclose(helper[i, :, :3], want_R[i], atol=1e-6)
        np.testing.assert_allclose(orc[i, :, :3], want_R[i], atol=1e-6)
        np.testing.assert_allclose(helper[i, :, 3], want_t, atol=1e-6)
        np.testing.assert_allclose(orc[i, :, 3], want_t, atol=1e-6)
    np.testing.assert_allclose(orc, helper, atol=1e-6)


def list_shape(P, shape):
    """(ctrl, m, reg, first, second) of P with the control lists or the correspondence list in one of the shapes the
    GPU edge tests run."""
    ctrl, m, reg = P["ctrl"], P["m"], P["reg"]
    first, second = corr_of(P)
    off, idx, val = (np.asarray(a) for a in ctrl)
    n = off.shape[0] - 1
    lists = [(list(idx[off[i]:off[i + 1]]), list(val[off[i]:off[i + 1]])) for i in range(n)]
    rng = np.random.default_rng(9)
    if shape == "dups":
        return with_duplicates(ctrl), m, reg, first, second
    if shape == "multi-pair":  # 1-3 pairs per point, one exact duplicate, shuffled across points
        import oracle

        idx3, _, cnt3 = oracle.BruteKnn(P["dst"]).neighborhoods(P["src"], 3, 0.02 ** 2)
        k = np.minimum(rng.integers(1, 4, n), cnt3)
        f = [idx3[i, j] for i in range(n) for j in range(k[i])]
        s = [i for i in range(n) for j in range(k[i])]
        f.append(f[0])
        s.append(s[0])
        o = rng.permutation(len(s))
        return ctrl, m, reg, np.array(f, np.int64)[o], np.array(s, np.int64)[o]
    if shape == "ragged":  # K from 0 to the full list, every third list empty
        for i in range(n):
            k = 0 if i % 3 == 0 else int(rng.integers(1, len(lists[i][0]) + 1))
            lists[i] = (lists[i][0][:k], lists[i][1][:k])
    elif shape == "hub":  # node 0 last in every list, as heavy as the list's first node
        lists = [(li + [0], lv + lv[:1]) for li, lv in lists]
    elif shape == "m = 1":
        lists = [([0], [float(np.sum((P["src"][i] - P["nodes"][0]) ** 2))]) for i in range(n)]
        m, reg = 1, (np.zeros(2, np.uint64), np.zeros(0, np.int64), np.zeros(0, np.float32))
    elif shape == "W = 0":  # every fourth list too far for its weights: they underflow to 0 in float and double
        for i in range(0, n, 4):
            lists[i] = (lists[i][0], [1.0] * len(lists[i][1]))
    o = np.zeros(n + 1, np.uint64)
    o[1:] = np.cumsum([len(a) for a, _ in lists])
    c = (o, np.array(sum((a for a, _ in lists), []), np.int64), np.array(sum((b for _, b in lists), []), np.float32))
    return c, m, reg, first, second


@pytest.mark.parametrize("dups", [False, True])
def test_oracle_normal_equations_match_the_reference_layout(swf, case, dups):
    P = dict(case)
    if dups:
        P["ctrl"] = with_duplicates(P["ctrl"])
    first, second = corr_of(P)
    check_normal_equations(swf, P, first, second)


@pytest.mark.parametrize("shape", ["multi-pair", "ragged", "hub", "m = 1", "W = 0"])
def test_oracle_normal_equations_match_the_reference_layout_on_more_list_shapes(swf, case, shape):
    """The list shapes the GPU edge tests judge the device on: several pairs per point (with a duplicate, in no
    particular order), ragged and empty control lists, a hub node in every list, one node without arcs, and lists
    whose weights all underflow (W_i = 0) on matched points."""
    P = dict(case)
    P["ctrl"], P["m"], P["reg"], first, second = list_shape(P, shape)
    if shape == "W = 0":
        _, _, _, W = ref.sorted_lists(P["ctrl"], KW["ctrl_sigma"])
        assert (W == 0).sum() > 100 and np.isin(np.nonzero(W == 0)[0], second).sum() > 50
    if shape == "ragged":
        lens = np.diff(P["ctrl"][0].astype(np.int64))
        assert (lens == 0).sum() > 100 and lens.max() > lens[lens > 0].min()
    check_normal_equations(swf, P, first, second)


def check_normal_equations(swf, P, first, second):
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
