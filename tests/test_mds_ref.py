"""The numpy restatement of multidimensional scaling (mds_ref.py) against numpy.linalg.eigh of the explicitly formed
-1/2 J E J in float64, and its rules: the lower-triangle B of a non-symmetric matrix, nev and the argument rules, the
MultidimensionalScalingXf fallback, the magnitude order with the clamp, the sign rule and the eigengap rule."""
import numpy as np
import pytest

import mds_ref as mr


def _dense_b(e):
    n = e.shape[0]
    J = np.eye(n) - np.full((n, n), 1.0 / n)
    return -0.5 * J @ e @ J


@pytest.mark.parametrize("squared", [True, False])
def test_b_is_double_centering_on_symmetric_input(squared):
    rng = np.random.default_rng(1)
    dm = mr.points_distances(rng.standard_normal((40, 3)), squared=squared)
    e = mr.entries(dm, squared).astype(np.float64)
    assert np.allclose(mr.b_matrix(dm, squared), _dense_b(e), rtol=0, atol=1e-12 * np.abs(e).max())


def test_b_reads_the_lower_triangle_of_non_symmetric_input():
    rng = np.random.default_rng(2)
    e = rng.uniform(0, 5, (30, 30)).astype(np.float32)
    full = _dense_b(e.astype(np.float64))
    B = mr.b_matrix(e, True)
    low = np.tril_indices(30)
    assert np.allclose(B[low], full[low], atol=1e-12) and np.array_equal(B, B.T)
    assert not np.allclose(B, full)  # the upper triangle of -1/2 J E J is not used


def test_unsquared_entries_round_once_in_fp32():
    d = np.array([[0, 1.1], [1.1, 0]], np.float32)
    assert mr.entries(d, False)[0, 1] == np.float32(np.float32(1.1) * np.float32(1.1))


def test_nev_and_argument_rules():
    assert mr.nev_of(10, 3, False) == 3 and mr.nev_of(10, 3, True) == 4
    assert mr.nev_of(4, 3, True) == 3 and mr.nev_of(4, 3, False) == 3
    assert mr.nev_of(4, 4, False) is None and mr.nev_of(4, 0, False) is None and mr.nev_of(4, 4, True) is None
    assert mr.nev_of(2, 1, False) == 1 and mr.nev_of(1, 1, False) is None
    assert mr.nev_of(5, 0, True) == 1


def test_xf_fallback():
    assert mr.xf_args(10, 0, True) == (2, False)
    assert mr.xf_args(10, 10, True) == (2, False) and mr.xf_args(10, 9, True) == (9, True)


def test_magnitude_order_and_clamp():
    w = np.array([1.0, -3.0, 3.0, 2.0, -0.5])
    assert mr.magnitude_order(w) == [2, 1, 3, 0, 4]
    rng = np.random.default_rng(3)
    x = rng.standard_normal((50, 3)) * [3, 2, 1]
    y = rng.standard_normal((50, 1)) * 4.0
    dm = (mr.points_distances(x) - 3 * mr.points_distances(y)).astype(np.float32)
    r = mr.mds(dm, 3)
    assert r["all_eigenvalues"].min() < -np.abs(r["all_eigenvalues"]).max() * 0.99  # the leading one is negative
    assert r["eigenvalues"][0] == 0.0 and np.all(r["embedding"][:, 0] == 0.0) and r["eigenvalues"][1] > 0


def test_sign_rule():
    assert list(mr.sign_rule(np.array([0.1, -0.9, 0.3]))) == [-0.1, 0.9, -0.3]
    assert list(mr.sign_rule(np.array([-0.5, 0.5]))) == [0.5, -0.5]  # lowest index on ties


def test_eigengap_rule():
    assert mr.eigengap_dim([5, 4, 1, 0.5], 3) == 2
    assert mr.eigengap_dim([5, 1, 0.9, 0.5], 3) == 1
    assert mr.eigengap_dim([2, 2, 2], 7) == 7  # spread below epsilon
    assert mr.eigengap_dim([1.0, 1.0 + 1e-8], 4) == 4
    assert mr.eigengap_dim([np.nan, 1.0], 3) == 3
    assert mr.eigengap_dim([3.0], 2) == 2


@pytest.mark.parametrize("n,max_dim", [(5, 2), (60, 3), (200, 1)])
def test_restatement_against_eigh(n, max_dim):
    """Eigenvalues are eigh's of -1/2 J E J by descending magnitude (clamped), and the embedding reproduces B's
    rank-dim part: X X^T = V diag(lambda) V^T."""
    rng = np.random.default_rng(n)
    dm = mr.points_distances(rng.standard_normal((n, 4)) * [4, 3, 2, 1])
    r = mr.mds(dm, max_dim)
    w, V = np.linalg.eigh(_dense_b(dm.astype(np.float64)))
    idx = np.argsort(-np.abs(w))[:max_dim]
    assert np.allclose(r["eigenvalues"], np.maximum(w[idx], 0), rtol=1e-10, atol=1e-10 * np.abs(w).max())
    g = V[:, idx] @ np.diag(np.maximum(w[idx], 0)) @ V[:, idx].T
    x = r["embedding"]
    assert np.allclose(x @ x.T, g, atol=1e-6 * np.abs(g).max())
    for j in range(max_dim):
        v = r["vectors"][:, j]
        assert v[np.argmax(np.abs(v))] > 0
