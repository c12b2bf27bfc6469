"""Pins the numpy restatement of k-means (kmeans_features_ref.py) on the CPU: at several D, D = 3 included, it equals a
serial C++ restatement of the same contract compiled with -ffp-contract=off (tests/cpp/kmeans_features_serial.cpp),
assignment, sums and whole Lloyd runs. At D = 3 test_kmeans_ransac_ref.py also pins it against the oracle."""
import os

import numpy as np
import pytest

import cxx
import kmeans_features_ref as kf


def _same_f32(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


@pytest.fixture(scope="module")
def serial(tmp_path_factory):
    src = os.path.join(cxx.ROOT, "tests", "cpp", "kmeans_features_serial.cpp")
    return cxx.build(src, str(tmp_path_factory.mktemp("kf") / "kmeans_features_serial"),
                     ["-O2", "-ffp-contract=off", "-march=x86-64-v3"], link=False)


def _run_serial(exe, tmp_path, pts, cent0, max_iter, tol):
    """Runs the serial restatement on one case: (centroids, labels, iterations, first-assignment labels)."""
    n, D = pts.shape
    k = len(cent0)
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        np.array([n, D, k, max_iter], np.int64).tofile(f)
        np.array([tol], np.float32).tofile(f)
        np.ascontiguousarray(pts, np.float32).tofile(f)
        np.ascontiguousarray(cent0, np.float32).tofile(f)
    out = tmp_path / "out.bin"
    cxx.run(exe, inp, out)
    raw = np.fromfile(out, np.uint8)
    it = int(raw[:8].view(np.int64)[0])
    cent = raw[8:8 + 4 * k * D].view(np.float32).reshape(k, D)
    off = 8 + 4 * k * D
    labels = raw[off:off + 8 * n].view(np.int64)
    first = raw[off + 8 * n:off + 16 * n].view(np.int64)
    return cent, labels, it, first


@pytest.mark.parametrize("D", [1, 2, 3, 6, 17, 64])
@pytest.mark.parametrize("case", list(kf.lloyd_cases(2)))
def test_restatement_equals_serial_cpp(serial, tmp_path, D, case):
    pts, cent0, max_iter, tol = kf.lloyd_cases(D)[case]
    oc, ol, oit, ofirst = _run_serial(serial, tmp_path, pts, cent0, max_iter, tol)
    fc, fl, fit = kf.lloyd(pts, cent0, max_iter, tol)
    assert fit == oit and np.array_equal(fl, ol) and _same_f32(fc, oc)
    if max_iter > 0:
        assert np.array_equal(ofirst, kf.assign(pts, cent0))


@pytest.mark.parametrize("D", [4, 33])
def test_restatement_equals_serial_cpp_on_non_dyadic_rows(serial, tmp_path, D):
    """Uniform floats and non-finite rows: the assignment and the first iteration's distances are exact in both."""
    rng = np.random.default_rng(D)
    pts = rng.standard_normal((3000, D)).astype(np.float32)
    pts[::211, D // 2] = np.nan
    pts[5::307, 0] = np.inf
    cent0 = rng.standard_normal((40, D)).astype(np.float32)
    _, _, _, ofirst = _run_serial(serial, tmp_path, pts, cent0, 1, 0.0)
    assert np.array_equal(ofirst, kf.assign(pts, cent0))
