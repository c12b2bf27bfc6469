"""The vectorised float64 normal equations of tests/warp_field_ref.py (the yardstick of the large device warp-field
cases) against the loop statements of tests/test_oracle_warp_field.py: the sparse Jacobian J in the reference's
equation order (J^T J, J^T b) and the dense block-by-block matrix, and against the arc rule itself."""
import numpy as np
import pytest

import test_oracle_warp_field as st
import warp_field_ref


@pytest.fixture(scope="module")
def wf(orc):
    from oracle import warp_field

    return warp_field


HUBER = float(np.float32(1e-2))


def arc_diffs(sysd, x):
    return (x[sysd["lo"]] - x[sysd["hi"]]).reshape(-1)


@pytest.mark.parametrize("w_pt,w_pl", [(0.1, 1.0), (1.0, 0.0), (0.0, 1.0)])
@pytest.mark.parametrize("x_scale", [0.0, 0.02])
def test_matches_the_sparse_jacobian(wf, w_pt, w_pl, x_scale):
    dst, nrm, src, first, second, nbhd = st.case(seed=11)
    n = src.shape[0]
    x = np.random.default_rng(5).normal(0, x_scale, (n, 6))
    kw = dict(w_pt=w_pt, w_pl=w_pl, stiffness=200.0, huber_delta=HUBER, reg_sigma=0.03)
    sysd = wf.system(dst, nrm, src, first, second, nbhd, x, **kw)
    S = warp_field_ref.NormalSystem(sysd)
    if x_scale:  # the regularisation differences fall on both sides of the Huber boundary
        d = np.abs(arc_diffs(sysd, x))
        assert (d > HUBER).sum() > 50 and (d < HUBER).sum() > 50
    J, b = st.jacobian(dst, nrm, src, first, second, nbhd, x, w_pt, w_pl, 200.0, HUBER, 0.03)
    A_ref, g_ref = (J.T @ J).toarray(), J.T @ b
    scale = np.abs(A_ref).max()
    A = S.matrix().toarray()
    assert np.abs(A - A_ref).max() <= 1e-12 * scale
    assert np.abs(S.g - g_ref).max() <= 1e-12 * np.abs(g_ref).max()
    v = np.random.default_rng(6).normal(0, 1, 6 * n)
    assert np.abs(S.matvec(v) - A_ref @ v).max() <= 1e-12 * scale * np.abs(v).sum()
    # the true residual of the exact solution is at the float64 floor, that of zero is 1
    sol = np.linalg.solve(A_ref, g_ref)
    assert S.true_rel_residual(sol) < 1e-9
    assert S.true_rel_residual(np.zeros(6 * n)) == pytest.approx(1.0)


def test_matches_the_dense_block_matrix(wf):
    dst, nrm, src, first, second, nbhd = st.case(n=80, seed=12, k=7)
    n = src.shape[0]
    x = np.random.default_rng(2).normal(0, 0.01, (n, 6))
    sysd = wf.system(dst, nrm, src, first, second, nbhd, x, w_pt=0.1, w_pl=1.0, stiffness=50.0, huber_delta=HUBER,
                     reg_sigma=0.02)
    S = warp_field_ref.NormalSystem(sysd)
    A_full = st.full_normal_matrix(sysd, n)
    A = S.matrix().toarray()
    assert np.abs(A - A_full).max() <= 1e-13 * np.abs(A_full).max()
    assert np.allclose(np.diag(A), sysd["diag"].reshape(-1), rtol=1e-13, atol=0)
    v = np.random.default_rng(3).normal(0, 1, 6 * n)
    assert np.allclose(S.matvec(v), A_full @ v, rtol=1e-12, atol=1e-12 * np.abs(A_full).max())


def test_the_arc_rule(wf):
    """Arcs come only from the first entry of each list to the others; self-arcs are dropped; a repeated neighbour, a
    neighbour listed from both sides stay separate arcs, in list order; fewer lists than points is allowed."""
    dst, nrm, src, first, second, _ = st.case(n=12, seed=13, k=3)
    n = src.shape[0]
    lists = [[3, 0, 5], [3, 3, 7], [5, 3], [1, 2, 2, 2], [2], [], [9, 10, 11, 9], [11, 10], [4, 11, 6, 0, 8, 7, 1]]
    off = np.concatenate([[0], np.cumsum([len(li) for li in lists])]).astype(np.uint64)
    idx = np.array([v for li in lists for v in li], np.int64)
    val = np.linspace(1e-4, 9e-4, idx.shape[0]).astype(np.float32)
    nbhd = (off, idx, val)
    want = [(min(li[0], v), max(li[0], v), val[int(off[j]) + k + 1])
            for j, li in enumerate(lists) for k, v in enumerate(li[1:]) if v != li[0]]
    x = np.random.default_rng(4).normal(0, 0.02, (n, 6))
    kw = dict(w_pt=0.1, w_pl=1.0, stiffness=30.0, huber_delta=HUBER, reg_sigma=0.03)
    sysd = wf.system(dst, nrm, src, first, second, nbhd, x, **kw)
    assert sysd["lo"].tolist() == [w[0] for w in want] and sysd["hi"].tolist() == [w[1] for w in want]
    # the coupling of each arc is h'^2 of its own weight, even for repeated arcs
    w = np.sqrt(np.float32(30.0)) * np.sqrt(np.exp(wf.rbf_coeff(0.03) * np.array([w[2] for w in want], np.float64)))
    diff = x[sysd["lo"]] - x[sysd["hi"]]
    h = w[:, None] * np.vectorize(st.sqrt_huber_d)(diff, HUBER)
    assert np.allclose(sysd["arc_c"], h * h, rtol=1e-6)
    S = warp_field_ref.NormalSystem(sysd)
    J, b = st.jacobian(dst, nrm, src, first, second, nbhd, x, 0.1, 1.0, 30.0, HUBER, 0.03)
    A_ref = (J.T @ J).toarray()
    assert np.abs(S.matrix().toarray() - A_ref).max() <= 1e-12 * np.abs(A_ref).max()
    assert np.abs(S.g - J.T @ b).max() <= 1e-12 * np.abs(J.T @ b).max()
