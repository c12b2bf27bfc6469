"""Pins the numpy restatement of k-means and RANSAC scoring (kmeans_ransac_ref.py) against the oracle on the CPU.

On small dyadic inputs the oracle's fp32 serial sums are exact, so its Lloyd loop (the reference's) and the
restatement's float64 one must agree bit for bit, repairs and tol stops included. The oracle's RANSAC scan is the
reference's sqrt(x) <= thresh, which the restatement states independently."""
import numpy as np
import pytest

import kmeans_ransac_ref as kr


def _same_f32(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


@pytest.mark.parametrize("case", list(kr.lloyd_cases()))
def test_lloyd_restatement_equals_oracle_on_dyadic_inputs(orc, case):
    pts, cent0, max_iter, tol = kr.lloyd_cases()[case]
    oc, ol, oit = orc.kmeans(pts, cent0, max_iter=max_iter, tol=tol)
    rc, rl, rit = kr.kmeans_lloyd(pts, cent0, max_iter, tol)
    assert rit == oit
    assert np.array_equal(rl, ol)
    assert _same_f32(rc, oc)
    if case == "tol_stop":
        assert oit < max_iter
    if case == "max_iter_0":
        assert oit == 0 and _same_f32(rc, cent0) and not rl.any()


def test_assign_restatement_equals_oracle(orc):
    rng = np.random.default_rng(21)
    pts = kr.dyadic(rng, (3000, 3), 3.0)
    cent = np.vstack([kr.dyadic(rng, (300, 3), 3.0)] * 2)  # every point ties between j and j + 300
    want, _ = orc.kmeans_assign(pts, cent)
    got = kr.kmeans_assign(pts, cent)
    assert np.array_equal(got, want.astype(np.int64)) and got.max() < 300
    # a finite point whose every squared distance overflows keeps label 0
    big = np.array([[3e19, 0, 0], [-3e19, 3e19, 0]], np.float32)
    want, _ = orc.kmeans_assign(big, cent)
    assert not kr.kmeans_assign(big, cent).any() and not want.any()


@pytest.mark.parametrize("n", [1, 31, 1025])
def test_ransac_counts_restatement_equals_oracle(orc, n):
    dst, src = kr.ransac_edge_pairs(n, seed=n)
    T_h = kr.ransac_edge_hypotheses(40, seed=1)
    got = kr.ransac_counts(dst, src, T_h, kr.THRESHOLDS)
    for t, g in zip(kr.THRESHOLDS, got):
        assert np.array_equal(g, orc.ransac_score(dst, src, T_h, t)), t
    if n == 1025:
        # the regimes are populated: the thresholds separate them
        c = dict(zip(kr.THRESHOLDS, (int(g[0]) for g in got)))  # hypothesis 0 is the identity
        assert c[0.0] < c[1e-20] < c[0.01] < c[1.8446743e19] <= c[3e38] < c[np.inf] < n
        assert got[kr.THRESHOLDS.index(1.4e-45)][0] == c[0.0] and c[-1.0] == 0 and got[-1].max() == 0
