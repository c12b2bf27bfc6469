"""Pins the numpy restatement of the projective correspondence search (tests/projective_ref.py) against a serial C++
restatement of find_correspondences_ (correspondence_search_projective.hpp:156-209) and of pointsToIndexMap compiled
with -ffp-contract=off (tests/cpp/projective_serial.cpp): the index map filled in index order with a strict smaller-z
test, then one source point at a time, the transform, projection, llround and distance written out in C++. The device
is pinned against the numpy restatement (test_gpu_projective_icp.py)."""
import os
import struct

import numpy as np
import pytest

import cxx
import depth_images_ref as dimg
import icp_ref
import projective_ref as pref

F = np.float32


@pytest.fixture(scope="module")
def serial_exe(tmp_path_factory):
    src = os.path.join(cxx.ROOT, "tests", "cpp", "projective_serial.cpp")
    return cxx.build(src, str(tmp_path_factory.mktemp("proj") / "projective_serial"),
                     flags=("-O2", "-ffp-contract=off"), link=False)


def serial(exe, tmp_path, dst, src, T, K, w, h, E, max_d2):
    Ez = np.zeros(12, F) if E is None else np.asarray(E, F).reshape(12)
    blob = struct.pack("<QQQQif", dst.shape[0], src.shape[0], w, h, int(E is not None), float(F(max_d2)))
    blob += np.asarray(K, F).tobytes() + np.asarray(T, F).reshape(12).tobytes() + Ez.tobytes()
    blob += np.asarray(dst, F).tobytes() + np.asarray(src, F).tobytes()
    (tmp_path / "in").write_bytes(blob)
    cxx.run(exe, tmp_path / "in", tmp_path / "out")
    out = (tmp_path / "out").read_bytes()
    m = struct.unpack("<Q", out[:8])[0]
    rec = np.frombuffer(out[8:], np.dtype([("f", "<u8"), ("s", "<u8"), ("v", "<f4")]), count=m)
    return rec["f"].astype(np.int64), rec["s"].astype(np.int64), rec["v"].astype(F)


@pytest.mark.parametrize("seed", range(6))
def test_restatement_matches_serial(serial_exe, tmp_path, seed):
    rng = np.random.default_rng(seed)
    w, h = [(7, 5), (31, 7), (33, 9), (16, 12), (1, 1), (64, 48)][seed]
    if seed % 2:  # skew and a last row other than (0, 0, 1)
        K = np.array([[0.9 * w, 0.3, w / 2], [0, 0.8 * w, h / 2], [0.001, -0.002, 1.25]], F)
    else:
        K = np.array([[0.9 * w, 0, w / 2], [0, 0.9 * w, h / 2], [0, 0, 1]], F)
    E = dimg.pose(seed, 0.2, 0.1) if seed in (2, 3, 5) else None
    cam = np.stack([rng.uniform(-1, 1, 400), rng.uniform(-1, 1, 400), rng.uniform(-0.2, 2, 400)], 1).astype(F)
    cam[1::17, 2] = cam[0, 2]  # exact z ties
    dst = cam if E is None else icp_ref.apply_f32(E, cam)
    dst = np.vstack([dst, dst[::5], [[np.nan, 0, 1], [0, np.inf, 1]]]).astype(F)
    T = dimg.pose(seed + 10, 0.03, 0.02)
    src = (icp_ref.apply_f32(T, dst) + rng.normal(scale=0.01, size=dst.shape)).astype(F)
    src = np.vstack([src, [[np.nan, 1, 1], [0, 0, -1]]]).astype(F)
    for max_d2 in (F(1e-3), F(0.05), F(np.inf)):
        f, s, v = pref.correspondences(dst, src, T, K, w, h, E, max_d2)
        wf, ws, wv = serial(serial_exe, tmp_path, dst, src, T, K, w, h, E, max_d2)
        assert f.size > 0 or w * h == 1
        assert np.array_equal(f, wf) and np.array_equal(s, ws)
        assert np.array_equal(v.view(np.uint32), wv.view(np.uint32))


def test_fraction_keeps_the_smallest_values_in_list_order():
    dst = np.array([[0, 0, 1], [0.5, 0, 1], [1, 0, 1], [1.5, 0, 1], [2, 0, 1]], F)
    src = np.array([[0.01, 0, 1], [0.51, 0, 1], [1.02, 0, 1], [1.51, 0, 1], [2.0, 0, 1]], F)
    K = np.array([[2, 0, 0], [0, 2, 0], [0, 0, 1]], F)
    T = icp_ref.identity().astype(F)
    f1, s1, v1 = pref.correspondences(dst, src, T, K, 5, 1, None, F(1.0))
    assert s1.tolist() == [0, 1, 2, 3, 4]
    for fraction, keep in ((0.5, 3), (0.3, 2), (0.99, 5), (0.05, 0)):
        f, s, v = pref.correspondences(dst, src, T, K, 5, 1, None, F(1.0), fraction)
        want = sorted(range(5), key=lambda k: v1[k])[:keep]  # a stable sort: ties keep the list order
        assert s.tolist() == want
