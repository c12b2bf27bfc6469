"""cb_solve_sym_eigen (host only, fp64 Householder + implicit QL) against numpy.linalg.eigh: eigenvalues within
1e-6 max|lambda|, orthonormal columns within 4 sqrt(D) 2^-24, det E > 0, the sign rule and NaN input."""
import numpy as np
import pytest

DIMS = [1, 2, 3, 4, 7, 16, 64, 257, 512]
KINDS = ["random", "diagonal", "repeated", "zero", "rank1", "graded"]


def _matrix(kind, D, rng):
    if kind == "random":
        A = rng.standard_normal((D, D))
        return A @ A.T / D
    if kind == "diagonal":
        return np.diag(rng.uniform(-3, 3, D))
    if kind == "repeated":
        Q = np.linalg.qr(rng.standard_normal((D, D)))[0]
        w = np.repeat([2.0, 1.0, -0.5], (D + 2) // 3)[:D]
        return (Q * w) @ Q.T
    if kind == "zero":
        return np.zeros((D, D))
    if kind == "rank1":
        v = rng.standard_normal(D)
        return np.outer(v, v)
    if kind == "graded":
        g = 10.0 ** np.linspace(0, -12, D)
        A = rng.standard_normal((D, D))
        return (A @ A.T / D) * np.outer(g, g)
    raise ValueError(kind)


def _check(cb, A):
    D = A.shape[0]
    A = A.astype(np.float32).astype(np.float64)  # the solver sees an fp32-rounded covariance
    A = np.triu(A) + np.triu(A, 1).T
    ev, E = cb.solve_sym_eigen(A)
    w = np.linalg.eigh(A)[0][::-1]
    lmax = max(np.abs(w).max(), np.finfo(np.float64).tiny)
    assert np.abs(ev.astype(np.float64) - w).max() <= 1e-6 * lmax, (ev, w)
    assert np.all(np.diff(ev) <= 0)
    E64 = E.astype(np.float64)
    assert np.abs(E64.T @ E64 - np.eye(D)).max() <= 4 * np.sqrt(D) * 2.0 ** -24
    assert np.linalg.det(E64) > 0
    for j in range(D - 1):  # the largest magnitude is a positive component (the last column may be negated for det)
        assert E64[:, j].max() >= np.abs(E64[:, j]).max(), j


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("scale", [1.0, 1e-30, 1e30])
def test_sym_eigen_against_eigh(cb, D, kind, scale):
    rng = np.random.default_rng(D * 7 + KINDS.index(kind))
    _check(cb, _matrix(kind, D, rng) * scale)


@pytest.mark.parametrize("D", [1, 4, 33])
def test_sym_eigen_nan_input(cb, D):
    A = np.eye(D)
    A[D // 2, D - 1] = A[D - 1, D // 2] = np.nan
    ev, E = cb.solve_sym_eigen(A)
    assert np.isnan(ev).all() and np.isnan(E).all()
    A[D // 2, D - 1] = A[D - 1, D // 2] = np.inf
    ev, E = cb.solve_sym_eigen(A)
    assert np.isnan(ev).all() and np.isnan(E).all()


def test_sym_eigen_sign_rule_on_ties(cb):
    """An exact tie of largest magnitudes in a column that is not the last: the lowest index is made positive. The
    eigenvectors of this matrix are (1, 1, 0)/sqrt2 (3), (1, -1, 0)/sqrt2 (1) and (0, 0, 1) (0.5); the solver's rotation
    for the 2 x 2 block has c = s exactly, so the middle column is (s, -c, 0) under the rule and would be (-s, c, 0)
    under a highest-index rule. The frame is then left-handed, so the last column is negated."""
    A = np.array([[2.0, 1.0, 0.0], [1.0, 2.0, 0.0], [0.0, 0.0, 0.5]])
    ev, E = cb.solve_sym_eigen(A)
    assert np.allclose(ev, [3, 1, 0.5])
    assert E[0, 1] == -E[1, 1] and E[0, 1] > 0 and E[2, 1] == 0
    assert E[0, 0] == E[1, 0] > 0
    assert E[2, 2] == -1.0 and np.linalg.det(E.astype(np.float64)) > 0


def test_sym_eigen_rejects_bad_arguments(cb):
    import ctypes as C
    assert cb.lib().cb_solve_sym_eigen(None, C.c_int(3), None, None) < 0
    A, ev, E = np.eye(2), np.empty(2, np.float32), np.empty((2, 2), np.float32)
    assert cb.lib().cb_solve_sym_eigen(cb._p(A), C.c_int(0), cb._p(ev), cb._p(E)) < 0
    assert cb.lib().cb_solve_sym_eigen(cb._p(A), C.c_int(2), cb._p(ev), cb._p(E)) == 1  # solved
    A[0, 1] = np.nan
    assert cb.lib().cb_solve_sym_eigen(cb._p(A), C.c_int(2), cb._p(ev), cb._p(E)) == 0  # non-finite input
