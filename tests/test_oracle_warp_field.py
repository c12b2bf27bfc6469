"""The dense warp-field oracle (oracle/warp_field_oracle.cpp) against an independent numpy / scipy statement of
estimateDenseWarpFieldCombinedMetric (registration/warp_field_estimation.hpp:368-715): the sparse Jacobian in the
reference's equation order, its normal equations, the CG of Eigen::ConjugateGradient, and the edge rules."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from cilantro_b200 import synth


@pytest.fixture(scope="module")
def wf(orc):
    from oracle import warp_field

    return warp_field


def rx(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])


def ry(b):
    c, s = np.cos(b), np.sin(b)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def rz(c_):
    c, s = np.cos(c_), np.sin(c_)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])


def drot(a, b, c):
    """R = Rz(c) Ry(b) Rx(a) and its three partial derivatives (by differentiating each factor)."""
    dRx = np.array([[0, 0, 0], [0, -np.sin(a), -np.cos(a)], [0, np.cos(a), -np.sin(a)]])
    dRy = np.array([[-np.sin(b), 0, np.cos(b)], [0, 0, 0], [-np.cos(b), 0, -np.sin(b)]])
    dRz = np.array([[-np.sin(c), -np.cos(c), 0], [np.cos(c), -np.sin(c), 0], [0, 0, 0]])
    return (rz(c) @ ry(b) @ rx(a), rz(c) @ ry(b) @ dRx, rz(c) @ dRy @ rx(a), dRz @ ry(b) @ rx(a))


def sqrt_huber(x, d):
    return np.sqrt(d * (abs(x) - 0.5 * d)) if abs(x) > d else np.sqrt(0.5) * abs(x)


def sqrt_huber_d(x, d):
    v = d / (2.0 * np.sqrt(d * (abs(x) - 0.5 * d))) if abs(x) > d else np.sqrt(0.5)
    return -v if x < 0 else v


def jacobian(dst, nrm, src, first, second, nbhd, x, w_pt, w_pl, stiffness, huber, sigma):
    """J (= At^T) and b, rows in the reference's equation order: point-to-point (3 per pair), point-to-plane, then
    6 per regularisation arc in neighbourhood order."""
    n = src.shape[0]
    rows, cols, vals, b = [], [], [], []

    def row(entries, rhs):
        r = len(b)
        for c, v in entries:
            rows.append(r)
            cols.append(c)
            vals.append(v)
        b.append(rhs)

    dst, src, nrm = dst.astype(np.float64), src.astype(np.float64), None if nrm is None else nrm.astype(np.float64)
    terms = []
    for f, s in zip(first, second):
        R, Ra, Rb, Rc = drot(*x[s, :3])
        ts = dst[f] - (R @ src[s] + x[s, 3:])
        terms.append((f, s, ts, Ra @ src[s], Rb @ src[s], Rc @ src[s]))
    if len(first) and w_pt > 0:
        w = np.sqrt(float(np.float32(w_pt)))
        for f, s, ts, da, db, dc in terms:
            for r in range(3):
                row([(6 * s, da[r] * w), (6 * s + 1, db[r] * w), (6 * s + 2, dc[r] * w), (6 * s + 3 + r, w)], ts[r] * w)
    if len(first) and w_pl > 0:
        w = np.sqrt(float(np.float32(w_pl)))
        for f, s, ts, da, db, dc in terms:
            nn = nrm[f]
            row([(6 * s, nn @ da * w), (6 * s + 1, nn @ db * w), (6 * s + 2, nn @ dc * w)] +
                [(6 * s + 3 + k, nn[k] * w) for k in range(3)], nn @ ts * w)
    off, idx, val = nbhd
    coeff = float(np.float32(-0.5) / (np.float32(sigma) ** 2))
    for j in range(len(off) - 1):
        lst = idx[off[j]:off[j + 1]]
        for k in range(1, len(lst)):
            lo, hi = sorted((lst[0], lst[k]))
            w = np.sqrt(float(np.float32(stiffness))) * np.sqrt(np.exp(coeff * float(val[off[j] + k])))
            for u in range(6):
                diff = x[lo, u] - x[hi, u]
                h = w * sqrt_huber_d(diff, huber)
                row([(6 * lo + u, h), (6 * hi + u, -h)], -w * sqrt_huber(diff, huber))
    J = sp.csc_matrix((vals, (rows, cols)), shape=(len(b), 6 * n))
    return J, np.array(b)


def case(n=60, seed=0, k=5):
    import oracle

    P = synth.warp_pair(n, seed=seed, spacing=0.01)
    dst, nrm, src = P["dst"], P["dst_normals"], P["src"]
    idx, d2, cnt = oracle.BruteKnn(src).neighborhoods(src, k, 3.0e38)
    from cilantro_b200.capi import neighborhood_csr

    nbhd = neighborhood_csr(idx, d2, cnt)
    i1, d = oracle.BruteKnn(dst).query(src, 0.05 ** 2)
    second = np.nonzero(i1 >= 0)[0]
    return dst, nrm, src, i1[second], second, nbhd


def full_normal_matrix(sysd, n):
    A = np.zeros((6 * n, 6 * n))
    iu = np.triu_indices(6)
    for i in range(n):
        blk = np.zeros((6, 6))
        blk[iu] = sysd["B"][i]
        blk = blk + np.triu(blk, 1).T
        A[6 * i:6 * i + 6, 6 * i:6 * i + 6] += blk
    for e, (lo, hi) in enumerate(zip(sysd["lo"], sysd["hi"])):
        for u in range(6):
            c = sysd["arc_c"][e, u]
            A[6 * lo + u, 6 * lo + u] += c
            A[6 * hi + u, 6 * hi + u] += c
            A[6 * lo + u, 6 * hi + u] -= c
            A[6 * hi + u, 6 * lo + u] -= c
    return A


@pytest.mark.parametrize("w_pt,w_pl", [(0.1, 1.0), (1.0, 0.0), (0.0, 1.0)])
def test_normal_equations_match_the_sparse_statement(wf, w_pt, w_pl):
    dst, nrm, src, first, second, nbhd = case()
    n = src.shape[0]
    rng = np.random.default_rng(3)
    # unknowns on both sides of the Huber boundary (1e-2) so that both branches enter
    x = rng.normal(0, 0.02, (n, 6))
    kw = dict(w_pt=w_pt, w_pl=w_pl, stiffness=200.0, huber=float(np.float32(1e-2)), sigma=0.03)
    J, b = jacobian(dst, nrm, src, first, second, nbhd, x, **kw)
    A_ref, g_ref = (J.T @ J).toarray(), J.T @ b
    sysd = wf.system(dst, nrm, src, first, second, nbhd, x, w_pt=w_pt, w_pl=w_pl, stiffness=200.0, huber_delta=1e-2,
                     reg_sigma=0.03)
    A = full_normal_matrix(sysd, n)
    scale = np.abs(A_ref).max()
    assert np.abs(A - A_ref).max() <= 1e-12 * scale
    assert np.abs(sysd["g"].reshape(-1) - g_ref).max() <= 1e-12 * np.abs(g_ref).max()
    assert np.allclose(sysd["diag"].reshape(-1), np.diag(A_ref), rtol=1e-12, atol=1e-12 * scale)


def test_fp64_solve_matches_spsolve(wf):
    dst, nrm, src, first, second, nbhd = case(seed=1)
    n = src.shape[0]
    kw = dict(w_pt=0.1, w_pl=1.0, stiffness=200.0, huber=float(np.float32(1e-2)), sigma=0.03)
    J, b = jacobian(dst, nrm, src, first, second, nbhd, np.zeros((n, 6)), **kw)
    delta = spla.spsolve((J.T @ J).tocsc(), J.T @ b).reshape(n, 6)
    got = wf.solve(dst, nrm, src, first, second, nbhd, w_pt=0.1, w_pl=1.0, stiffness=200.0, huber_delta=1e-2,
                   reg_sigma=0.03, max_gn_iter=1, max_cg_iter=100000, cg_tol=1e-12, double=True)
    want = np.stack([np.hstack([drot(*d[:3])[0], d[3:, None]]) for d in delta])
    # the transforms are stored in float: agreement to float rounding of the solution
    assert np.abs(got["T"] - want).max() < 1e-6 * max(1.0, np.abs(want).max())
    assert got["gn_steps"] == 1 and got["cg_iterations"] > 0


def numpy_cg(A, b, tol, max_iter):
    """The CG of DESIGN §4.13 (Eigen::ConjugateGradient, diagonal preconditioner, zero guess), in float64."""
    x = np.zeros_like(b)
    rhs2 = b @ b
    if rhs2 == 0:
        return 0
    thr = max(tol * tol * rhs2, np.finfo(np.float32).tiny)
    r = b.copy()
    if r @ r < thr:
        return 0
    d = np.diag(A)
    inv = np.where(d != 0, 1.0 / np.where(d != 0, d, 1.0), 1.0)
    p = inv * r
    abs_new = r @ p
    i = 0
    while i < max_iter:
        q = A @ p
        alpha = abs_new / (p @ q)
        x += alpha * p
        r -= alpha * q
        if r @ r < thr:
            break
        z = inv * r
        abs_old, abs_new = abs_new, r @ z
        p = z + (abs_new / abs_old) * p
        i += 1
    return i


@pytest.mark.parametrize("seed,tol", [(2, 1e-5), (4, 1e-8), (5, 1e-3)])
def test_cg_iteration_count_matches_numpy_restatement(wf, seed, tol):
    # small, well-conditioned systems: the count must not hinge on the last bits of a long Krylov recurrence
    dst, nrm, src, first, second, nbhd = case(n=12, seed=seed, k=3)
    n = src.shape[0]
    kw = dict(w_pt=1.0, w_pl=1.0, stiffness=1.0, huber=float(np.float32(1e-2)), sigma=0.03)
    J, b = jacobian(dst, nrm, src, first, second, nbhd, np.zeros((n, 6)), **kw)
    want = numpy_cg((J.T @ J).toarray(), J.T @ b, tol, 10000)
    got = wf.solve(dst, nrm, src, first, second, nbhd, w_pt=1.0, w_pl=1.0, stiffness=1.0, huber_delta=1e-2,
                   reg_sigma=0.03, max_gn_iter=1, max_cg_iter=10000, cg_tol=tol, double=True)
    assert 0 < want < 6 * n
    assert got["cg_iterations"] == want


def test_sqrt_huber_loss_and_derivative(wf):
    d = 1e-2
    for x in (0.0, 0.5 * d, d, np.nextafter(np.float32(d), np.float32(1)), 3 * d, -0.5 * d, -3 * d):
        x32 = float(np.float32(x))
        assert wf.huber(x32, d) == pytest.approx(sqrt_huber(x32, float(np.float32(d))), rel=1e-6, abs=1e-12)
        assert wf.huber(x32, d, True) == pytest.approx(sqrt_huber_d(x32, float(np.float32(d))), rel=1e-6)
    assert wf.huber(0.0, d) == 0.0 and wf.huber(0.0, d, True) == pytest.approx(np.sqrt(0.5))
    # continuous across the boundary, and the derivative is the derivative of the loss
    for x in (0.5 * d, 2 * d, -2 * d):
        h = 1e-4 * d
        fd = (sqrt_huber(x + h, d) - sqrt_huber(x - h, d)) / (2 * h)
        assert wf.huber(x, d, True) == pytest.approx(fd, rel=1e-3)


def test_euler_parametrisation_jacobian(wf):
    rng = np.random.default_rng(7)
    for a, b, c in rng.uniform(-1.0, 1.0, (5, 3)):
        M, Ma, Mb, Mc = wf.rotation_terms(a, b, c)
        assert np.allclose(M.T, rz(c) @ ry(b) @ rx(a), atol=1e-14)  # rot_coeffs^T = Rz Ry Rx
        h = 1e-6
        for k, D in enumerate((Ma, Mb, Mc)):
            e = np.zeros(3)
            e[k] = h
            fd = (wf.rotation_terms(*(np.array([a, b, c]) + e))[0] - wf.rotation_terms(*(np.array([a, b, c]) - e))[0]) / (2 * h)
            assert np.abs(D - fd).max() < 1e-8


def identity_set(n):
    return np.tile(np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32), (n, 1, 1))


def test_edge_rules_give_identity_and_false(wf):
    dst, nrm, src, first, second, nbhd = case(n=30, seed=8)
    n = src.shape[0]
    empty = (np.zeros(n + 1, np.uint64), np.zeros(0, np.int64), np.zeros(0, np.float32))
    for kw in (dict(first=first[:0], second=second[:0], nbhd=nbhd, w_pt=0.1, w_pl=1.0),  # no correspondences
               dict(first=first, second=second, nbhd=nbhd, w_pt=0.0, w_pl=0.0)):        # no metric
        r = wf.solve(dst, nrm, src, **kw)
        assert not r["converged"] and r["gn_steps"] == 0
        assert np.array_equal(r["T"], identity_set(n))
    # empty neighbourhoods and self-arcs add no arcs: the same system as no regularisation at all
    self_arcs = (np.arange(n + 1, dtype=np.uint64) * 2, np.repeat(np.arange(n), 2), np.zeros(2 * n, np.float32))
    x = np.random.default_rng(1).normal(0, 0.01, (n, 6))
    ref = wf.system(dst, nrm, src, first, second, empty, x, w_pt=0.1)
    for nb in (self_arcs, (np.zeros(n + 1, np.uint64), np.zeros(0, np.int64), np.zeros(0, np.float32))):
        got = wf.system(dst, nrm, src, first, second, nb, x, w_pt=0.1)
        assert got["arc_c"].shape[0] == 0
        assert np.array_equal(got["B"], ref["B"]) and np.array_equal(got["g"], ref["g"])
    # a point without correspondence and arcs keeps the identity
    r = wf.solve(dst, nrm, src, first[1:], second[1:], empty, w_pt=0.1)
    assert np.array_equal(r["T"][second[0]], identity_set(1)[0])
