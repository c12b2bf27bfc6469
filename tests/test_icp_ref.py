"""tests/icp_ref.py, the float64 ICP step of the GPU edge tests, pinned against the product's host solves
(cb_solve_kabsch_moments, cb_solve_gauss_newton), so that a disagreement on the GPU points at the device, not at
the reference. No GPU needed."""
import numpy as np
import pytest

import icp_ref
from cilantro_b200 import synth
from conftest import frob


def _raw_moments(d, q):
    s = np.zeros(16)
    s[0] = len(d)
    s[1:4] = d.sum(0)
    s[4:7] = q.sum(0)
    s[7:16] = (d.T @ q).ravel()
    return s


@pytest.mark.parametrize("case", ["generic", "reflection", "planar", "thin"])
def test_kabsch_reference_matches_host_solve(cb, case):
    rng = np.random.default_rng({"generic": 1, "reflection": 2, "planar": 3, "thin": 4}[case])
    for _ in range(20):
        q = rng.normal(size=(200, 3)) * [3.0, 2.0, 1.0]  # distinct singular values: the reflection fix is well posed
        if case == "planar":
            q[:, 2] = 0.0
        if case == "thin":
            q[:, 2] *= 1e-3
        T = synth.rigid_from_axis_angle(rng.normal(size=3), rng.uniform(-2, 2), rng.normal(size=3))
        d = icp_ref.apply(T, q) + 1e-4 * rng.normal(size=q.shape)
        if case == "reflection":
            d[:, 2] = -d[:, 2]
        Tp, ok = cb.solve_kabsch_moments(_raw_moments(d, q))
        Tr, sigma = icp_ref.kabsch(d, q)
        assert ok
        # the branch helper agrees with what the product's matrices say about sigma
        assert icp_ref.polar_accepts(sigma) == (np.linalg.det(sigma) > 1e-6 * np.linalg.norm(sigma) ** 3)
        if case == "planar":
            assert not icp_ref.polar_accepts(sigma)
            # rank 2: the rotation is still unique (u2 = u0 x u1)
        assert frob(Tp, Tr) < 2e-5, (case, frob(Tp, Tr))
        assert case != "generic" or icp_ref.polar_accepts(sigma)


def test_polar_acceptance_helper_on_constructed_ratios():
    R = synth.rigid_from_axis_angle([1, 2, 3], 0.7, [0, 0, 0])[:, :3]
    for target in (1e-6 * (1 - 1e-2), 1e-6 * (1 + 1e-2)):
        # sigma = R diag(1, 1, e): det / |.|_F^3 = e / (2 + e^2)^1.5
        e = target * 2 ** 1.5
        for _ in range(4):
            e = target * (2 + e * e) ** 1.5
        sigma = R @ np.diag([1.0, 1.0, e])
        assert abs(icp_ref.det_ratio(sigma) / target - 1) < 1e-9
        assert icp_ref.polar_accepts(sigma) == (target > 1e-6)
    assert not icp_ref.polar_accepts(np.zeros((3, 3)))
    assert not icp_ref.polar_accepts(-np.eye(3))
    assert icp_ref.polar_accepts(np.eye(3))


@pytest.mark.parametrize("w_pt,w_pl,sym", [(0.0, 1.0, False), (0.3, 1.0, False), (1.0, 0.0, False), (0.1, 1.0, True)])
def test_gauss_newton_reference_matches_host_solve(cb, w_pt, w_pl, sym):
    dst, src, nrm, T_ref = synth.icp_pair(3000, seed=8, noise=0.0005, with_normals=True)
    src_n = (nrm.astype(np.float64) @ synth.invert(T_ref)[:, :3].T).astype(np.float32) if sym else None
    T = (0.7 * T_ref + 0.3 * icp_ref.identity()).astype(np.float32)
    idx = np.arange(3000)
    dm = dst.astype(np.float64).mean(0).astype(np.float32)
    sm = src.astype(np.float64).mean(0).astype(np.float32)
    Tn, info = icp_ref.combined_step(dst, nrm, src, T, idx, idx, w_pt, w_pl, dm, sm, src_n=src_n)
    # the same normal equations through the product's host solve (pivoted sums -> update -> un-centre -> finish)
    A, b = info["A"], info["b"]
    sums = np.zeros(28)
    sums[0] = 3000
    sums[1:22] = A[np.triu_indices(6)]
    sums[22:] = b
    Tgn, dn = cb.solve_gauss_newton(sums)
    assert dn > 0
    Tgn = Tgn.astype(np.float64)
    smt = icp_ref.apply_f32(T, sm[None])[0].astype(np.float64)
    Tgn[:, 3] = Tgn[:, 3] - Tgn[:, :3] @ smt + dm
    Tp = icp_ref.compose(np.hstack([cb.solve_rotation(Tgn[:, :3]), Tgn[:, 3:]]), T)
    assert frob(Tp, Tn) < 2e-6, frob(Tp, Tn)
    assert frob(Tn, T_ref) < frob(T, T_ref)  # and the step goes towards the generating pose


def test_normal_equations_match_explicit_eq_vecs():
    rng = np.random.default_rng(5)
    d, s = rng.normal(size=(50, 3)), rng.normal(size=(50, 3))
    n = rng.normal(size=(50, 3))
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    A, b = icp_ref.normal_equations(d, s, 0.4, 0.7, n)
    v, e = d + s, d - s
    A2, b2 = np.zeros((6, 6)), np.zeros(6)
    for i in range(50):
        vx = np.array([[0, -v[i, 2], v[i, 1]], [v[i, 2], 0, -v[i, 0]], [-v[i, 1], v[i, 0], 0]])
        E = np.vstack([vx, np.eye(3)])  # eq_vecs, transform_estimation.hpp:306-316
        a = np.concatenate([np.cross(v[i], n[i]), n[i]])
        A2 += 0.4 * E @ E.T + 0.7 * np.outer(a, a)
        b2 += 0.4 * E @ e[i] + 0.7 * a * (n[i] @ e[i])
    assert np.allclose(A, A2, rtol=1e-13, atol=1e-12) and np.allclose(b, b2, rtol=1e-13, atol=1e-12)
