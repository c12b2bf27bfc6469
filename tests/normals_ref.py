"""Float64 bounds on the eigen step of the normal estimation (sym3_smallest in sym3_eigen.cuh), applied per point to
the covariance the product returned, so that the reference is exact at every scale:

    from normals_ref import check_eigen
    worst = check_eigen(cov6, normals, curvature, "label")

Each point's (fp32) cov6 is solved with numpy.linalg.eigh in float64 (w ascending, w2 = max |w|, gap = (w1 - w0) / w2):
  - the normal is finite and unit to 1e-6; where gap >= GAP_CLEAR the sine of its angle to the eigenvector of w0 is
    below 1e-6 / gap, elsewhere (a near-degenerate smallest pair) the eigenspace residual |C n - w0 n| / w2 < 1e-6;
  - the curvature w0 / (w0 + w1 + w2) within 1e-6 w2 / w0 relative where w0 > 1e-5 w2, else within 1e-6 absolute;
  - a covariance with a NaN or infinite entry (fewer than 3 neighbours, or an overflowed sum) gives a NaN normal and
    curvature; the zero covariance gives the normal +-e_x (the solver's identity column) and a NaN curvature (0 / 0).
tests/test_solve_device.py::test_device_sym3_smallest holds the solver itself to the same bounds.
"""
import numpy as np

GAP_CLEAR = 1e-3


def full(c6):
    c6 = np.asarray(c6, np.float64)
    return np.stack([c6[:, [0, 1, 2]], c6[:, [1, 3, 4]], c6[:, [2, 4, 5]]], axis=1)


def check_eigen(cov6, normals, curvature, label=""):
    """Asserts the bounds above on every point; returns the worst ratio of error to bound per quantity, with the point
    counts of each class."""
    cov6 = np.asarray(cov6, np.float32).reshape(-1, 6)
    nrm = np.asarray(normals, np.float32).reshape(-1, 3)
    curv = np.asarray(curvature, np.float32).reshape(-1)
    bad = ~np.isfinite(cov6).all(axis=1)
    assert np.array_equal(np.isnan(nrm).any(axis=1), bad), (label, "normal NaN pattern")
    assert np.isnan(nrm[bad]).all() and np.isnan(curv[bad]).all(), (label, "non-finite covariance")
    zero = ~bad & (cov6 == 0).all(axis=1)
    ex = np.abs(nrm[zero])
    assert np.array_equal(ex, np.tile(np.float32([1, 0, 0]), (len(ex), 1))), (label, "zero covariance normal")
    assert np.isnan(curv[zero]).all(), (label, "zero covariance curvature")
    ok = ~bad & ~zero
    worst = {"points": int(ok.sum()), "non-finite": int(bad.sum()), "zero": int(zero.sum()),
             "sin*gap/1e-6": 0.0, "residual/1e-6": 0.0, "curvature err/bound": 0.0}
    if not ok.any():
        return worst
    assert np.isfinite(nrm[ok]).all() and not np.isnan(curv[ok]).any(), (label, "finite covariance, NaN output")
    C = full(cov6[ok])
    w, V = np.linalg.eigh(C)
    n = nrm[ok].astype(np.float64)
    norm = np.linalg.norm(n, axis=1)
    assert np.all(np.abs(norm - 1) < 1e-6), (label, "unit", np.abs(norm - 1).max())
    w2 = np.abs(w).max(axis=1)
    gap = (w[:, 1] - w[:, 0]) / w2
    clear = gap >= GAP_CLEAR
    sin = np.linalg.norm(np.cross(n, V[:, :, 0]), axis=1) / norm
    r_sin = sin * gap / 1e-6
    res = np.linalg.norm(np.einsum("pij,pj->pi", C, n) - w[:, :1] * n, axis=1) / w2
    r_res = res / 1e-6
    r_n = np.where(clear, r_sin, r_res)
    i = int(np.argmax(r_n))
    assert r_n[i] < 1, (label, "normal", "sin" if clear[i] else "residual", sin[i], res[i], gap[i], cov6[ok][i], n[i])
    c = curv[ok].astype(np.float64)
    rel = w[:, 0] > 1e-5 * w2
    with np.errstate(divide="ignore", invalid="ignore"):
        kr = w[:, 0] / w.sum(axis=1)
        err = np.where(c == kr, 0.0, np.abs(c - kr))  # (equal infinities: an indefinite matrix with trace 0)
    r_c = np.where(rel, err / np.where(rel, kr, 1.0) / (1e-6 * w2 / np.where(rel, w[:, 0], 1.0)), err / 1e-6)
    j = int(np.argmax(r_c))
    assert r_c[j] < 1, (label, "curvature", c[j], kr[j], w[j], cov6[ok][j])
    worst["sin*gap/1e-6"] = float(r_sin[clear].max()) if clear.any() else 0.0
    worst["residual/1e-6"] = float(r_res[~clear].max()) if (~clear).any() else 0.0
    worst["curvature err/bound"] = float(r_c.max())
    return worst


def merge(into, worst):
    """Running maxima of check_eigen's ratios (counts add up)."""
    for key, v in worst.items():
        into[key] = into.get(key, 0) + v if isinstance(v, int) else max(into.get(key, 0.0), v)
    return into


def fmt(worst):
    return ", ".join(f"{k} {v}" if isinstance(v, int) else f"{k} {v:.3g}" for k, v in worst.items())
