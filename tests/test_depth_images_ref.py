"""The numpy restatement of the depth-image <-> cloud contract (tests/depth_images_ref.py, DESIGN §4.20) equals a serial
C++ restatement of the reference's loops compiled with -ffp-contract=off (tests/cpp/depth_images_serial.cpp) bit for
bit: the 3 x 3 inverse, back-projection in both extrinsics associations, normals, compaction, colours, and the serial
z-buffer with its tie and range rules. The device is pinned against the numpy restatement (test_gpu_depth_images.py)."""
import os
import struct

import numpy as np
import pytest

import cxx
import depth_images_ref as ref


@pytest.fixture(scope="module")
def serial(tmp_path_factory):
    src = os.path.join(cxx.ROOT, "tests", "cpp", "depth_images_serial.cpp")
    return cxx.build(src, str(tmp_path_factory.mktemp("di") / "depth_images_serial"),
                     flags=("-O2", "-ffp-contract=off"), link=False)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def run_back(serial, tmp_path, depth, K, scale, max_depth, rgb, T, normals, keep_invalid):
    h, w = depth.shape
    f32 = depth.dtype == np.float32
    hdr = struct.pack("<QQiiff", w, h, int(f32), int(max_depth is not None), scale,
                      0.0 if max_depth is None else max_depth)
    Tz = np.zeros(12, np.float32) if T is None else np.asarray(T, np.float32).reshape(12)
    blob = hdr + np.asarray(K, np.float32).tobytes() + struct.pack("<i", int(T is not None)) + Tz.tobytes()
    blob += struct.pack("<iii", int(normals), int(keep_invalid), int(rgb is not None)) + depth.tobytes()
    if rgb is not None:
        blob += rgb.tobytes()
    (tmp_path / "in").write_bytes(blob)
    cxx.run(serial, "back", tmp_path / "in", tmp_path / "out")
    out = (tmp_path / "out").read_bytes()
    m = struct.unpack("<Q", out[:8])[0]
    arr = np.frombuffer(out[8:], np.float32)
    p = arr[:3 * m].reshape(m, 3)
    rest = arr[3 * m:]
    n = rest[:3 * m].reshape(m, 3) if normals else None
    rest = rest[3 * m:] if normals else rest
    c = rest[:3 * m].reshape(m, 3) if rgb is not None else None
    return p, n, c


def run_render(serial, tmp_path, pts, K, w, h, mode, scale, max_depth, T, colors):
    n = pts.shape[0]
    blob = struct.pack("<QQQiiff", n, w, h, mode, int(max_depth is not None), scale,
                       0.0 if max_depth is None else max_depth)
    Tz = np.zeros(12, np.float32) if T is None else np.asarray(T, np.float32).reshape(12)
    blob += np.asarray(K, np.float32).tobytes() + struct.pack("<i", int(T is not None)) + Tz.tobytes()
    blob += struct.pack("<i", int(colors is not None)) + pts.astype(np.float32).tobytes()
    if colors is not None:
        blob += colors.astype(np.float32).tobytes()
    (tmp_path / "in").write_bytes(blob)
    cxx.run(serial, "render", tmp_path / "in", tmp_path / "out")
    out = (tmp_path / "out").read_bytes()
    if mode == 2:
        return np.frombuffer(out, np.uint64).reshape(h, w)
    dt = np.uint16 if mode == 0 else np.float32
    nb = w * h * np.dtype(dt).itemsize
    d = np.frombuffer(out[:nb], dt).reshape(h, w)
    return d if colors is None else (d, np.frombuffer(out[nb:], np.uint8).reshape(h, w, 3))


def test_inverse_matches_eigen_order():
    # the restated inverse is within rounding of float64's, for the pinhole and the general K
    for K in (ref.K_PINHOLE, ref.K_GENERAL):
        Ki = ref.inverse3(K)
        assert np.allclose(Ki, np.linalg.inv(K.astype(np.float64)), rtol=1e-5, atol=1e-8)


@pytest.mark.parametrize("dtype", [np.uint16, np.float32])
@pytest.mark.parametrize("kind", ["full", "holed", "special", "single", "zero"])
@pytest.mark.parametrize("wh", [(1, 1), (7, 1), (1, 9), (3, 3), (37, 11)])
def test_back_projection_equals_serial(serial, tmp_path, dtype, kind, wh):
    w, h = wh
    depth = ref.frame(kind, w, h, dtype, seed=w * 31 + h)
    rgb = ref.rgb_frame(w, h)
    T = ref.pose(5)
    for K in (ref.K_PINHOLE, ref.K_GENERAL):
        for scale, max_depth in ((1000.0, None), (1000.0, 1.6), (0.5, None)):
            for normals in (False, True):
                for keep in (False, True):
                    for ext in (None, T):
                        col = rgb if normals == keep else None
                        got = ref.depth_to_points(depth, K, scale, max_depth, col, ext, normals, keep)
                        want = run_back(serial, tmp_path, depth, K, scale, max_depth, col, ext, normals, keep)
                        for g, e in zip(got, want):
                            assert (g is None) == (e is None)
                            if g is not None:
                                assert np.array_equal(bits(g), bits(e)), (K, scale, max_depth, normals, keep, ext)


def test_zero_cross_product_keeps_a_zero_normal(serial, tmp_path):
    # depths of 1e-25: every cross-product term underflows to zero, so the normal is the zero vector, kept as it is
    depth = np.full((4, 5), 1e-25, np.float32)
    p, n, _ = ref.depth_to_points(depth, ref.K_PINHOLE, 1.0, None, None, None, True, False)
    assert p.shape == (6, 3) and np.all(n == 0)
    sp, sn, _ = run_back(serial, tmp_path, depth, ref.K_PINHOLE, 1.0, None, None, None, True, False)
    assert np.array_equal(bits(n), bits(sn)) and np.array_equal(bits(p), bits(sp))


def render_points(seed, n=3000):
    """Points in front of, behind and beside a 40 x 30 camera, at half-pixel projections, non-finite, out of the raw
    range, and many per pixel with exact raw-depth ties."""
    rng = np.random.default_rng(seed)
    p = np.empty((n, 3), np.float32)
    z = rng.uniform(-0.5, 3.0, n)
    u = rng.uniform(-5, 45, n)
    v = rng.uniform(-5, 35, n)
    u[: n // 10] = np.round(u[: n // 10]) + 0.5  # half-pixel projections (exact for z = 1)
    z[: n // 10] = 1.0
    z[n // 10: n // 5] = np.round(z[n // 10: n // 5] * 4) / 4  # exact raw-depth ties
    u[n // 10: n // 5] = np.round(u[n // 10: n // 5] / 4)
    v[n // 10: n // 5] = np.round(v[n // 10: n // 5] / 4)
    p[:, 0] = (u - 20.0) * z / 40.0
    p[:, 1] = (v - 15.0) * z / 40.0
    p[:, 2] = z
    p[-5:] = [[np.nan, 0, 1], [0, np.inf, 1], [0, 0, np.inf], [0, 0, 70.0], [0, 0, np.nan]]
    return p


K_RENDER = np.array([[40.0, 0.0, 20.0], [0.0, 40.0, 15.0], [0.0, 0.0, 1.0]], np.float32)


@pytest.mark.parametrize("seed", [0, 1])
def test_render_equals_serial(serial, tmp_path, seed):
    pts = render_points(seed)
    col = np.random.default_rng(seed).uniform(-0.2, 1.2, pts.shape).astype(np.float32)
    col[0] = np.nan
    T = ref.pose(seed + 7, angle=0.05, shift=0.05)
    w, h = 40, 30
    for ext in (None, T):
        for K in (K_RENDER, ref.K_GENERAL):
            got = ref.points_to_index_map(pts, K, w, h, ext)
            assert np.array_equal(got, run_render(serial, tmp_path, pts, K, w, h, 2, 1.0, None, ext, None))
            for mode, dt in ((0, np.uint16), (1, np.float32)):
                for scale, md in ((1000.0, None), (1000.0, 2.0), (30000.0, None)):
                    for c in (None, col):
                        g = ref.points_to_depth_image(pts, K, w, h, dt, scale, md, c, ext)
                        e = run_render(serial, tmp_path, pts, K, w, h, mode, scale, md, ext, c)
                        if c is None:
                            assert np.array_equal(g.view(np.uint8), e.view(np.uint8)), (mode, scale, md)
                        else:
                            assert np.array_equal(g[0].view(np.uint8), e[0].view(np.uint8)), (mode, scale, md)
                            assert np.array_equal(g[1], e[1])
