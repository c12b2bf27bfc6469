"""Pins the numpy restatement of the PCA projection and reconstruction folds (pca_features_ref.py) on the CPU: at
several D and k it equals a serial C++ restatement of the same contract compiled with -ffp-contract=off
(tests/cpp/pca_features_serial.cpp), bit for bit; and its float64 covariance keeps the reference's per-dimension
non-finite semantics and sample-size expressions."""
import os

import numpy as np
import pytest

import cxx
import pca_features_ref as pf


def _same_f32(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


@pytest.fixture(scope="module")
def serial(tmp_path_factory):
    src = os.path.join(cxx.ROOT, "tests", "cpp", "pca_features_serial.cpp")
    return cxx.build(src, str(tmp_path_factory.mktemp("pf") / "pca_features_serial"),
                     ["-O2", "-ffp-contract=off", "-march=x86-64-v3"], link=False)


@pytest.mark.parametrize("D,k", [(1, 1), (2, 1), (5, 5), (6, 3), (17, 4), (33, 33), (130, 9)])
def test_folds_equal_serial_cpp(serial, tmp_path, D, k):
    rng = np.random.default_rng(D * 100 + k)
    n = 257
    rows = (rng.standard_normal((n, D)) * rng.uniform(0.1, 100, D) + rng.uniform(-1e3, 1e3, D)).astype(np.float32)
    rows[7, D // 2] = np.nan
    mean = rows[8:].mean(0).astype(np.float32)
    E = np.linalg.qr(rng.standard_normal((D, D)))[0].astype(np.float32)
    q = rng.standard_normal((n, k)).astype(np.float32)
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        np.array([n, D, k], np.int64).tofile(f)
        for a in (rows, mean, E, q):
            np.ascontiguousarray(a, np.float32).tofile(f)
    out = tmp_path / "out.bin"
    cxx.run(serial, inp, out)
    raw = np.fromfile(out, np.float32)
    proj, rec = raw[:n * k].reshape(n, k), raw[n * k:].reshape(n, D)
    assert _same_f32(pf.project(rows, mean, E, k), proj)
    assert _same_f32(pf.reconstruct(q, mean, E), rec)


def test_mean_cov_nonfinite_rule():
    rows = np.random.default_rng(3).standard_normal((50, 5)).astype(np.float32)
    rows[4, 1] = np.nan
    rows[9, 3] = np.inf
    rows[10, 4], rows[11, 4] = np.inf, -np.inf
    mean, cov, ok = pf.mean_cov(rows)
    assert ok
    assert np.isnan(mean[1]) and mean[3] == np.inf and np.isnan(mean[4]) and np.isfinite(mean[[0, 2]]).all()
    bad = [1, 3, 4]
    assert np.isnan(cov[bad, :]).all() and np.isnan(cov[:, bad]).all()
    good = np.ix_([0, 2], [0, 2])
    ref = np.cov(rows[:, [0, 2]].astype(np.float64).T)
    assert np.allclose(cov[good], ref, rtol=1e-14, atol=0)


def test_mean_cov_sample_size_expressions():
    rows = np.arange(12, dtype=np.float32).reshape(3, 4)
    m, c, ok = pf.mean_cov(rows[:1], min_sample_size=2)
    assert not ok and np.isnan(m).all() and np.isnan(c).all()
    m, c, ok = pf.mean_cov(rows[:1], min_sample_size=1)
    assert ok and np.array_equal(m, rows[0]) and np.isnan(c).all()
    m, c, ok = pf.mean_cov(rows[:0], min_sample_size=0)
    assert ok and np.isnan(m).all() and (c == 0).all() and np.signbit(c).all()
    m, c, ok = pf.mean_cov(rows, subset=[], min_sample_size=0)
    assert ok and np.isnan(m).all() and (c == 0).all() and not np.signbit(c).any()
