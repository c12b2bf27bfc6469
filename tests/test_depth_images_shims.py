"""The C++ drop-ins of core/image_point_cloud_conversions.hpp (the converters, depthImageToPoints…,
pointsToDepthImage, pointsColorsToRGBDImages, pointsToIndexMap) and PointCloud3f's image constructors: the headers and
the example compile with and without Eigen, double MetricDepth is a compile-time error, the existing PointCloud3f
constructors stay unambiguous, and on the GPU the shim program gives the C ABI's results bit for bit and the example
registers its two rendered frames."""
import os

import numpy as np
import pytest

import cxx
import depth_images_ref as ref

ROOT = cxx.ROOT
SHIM = os.path.join(ROOT, "tests", "cpp", "test_depth_images_shim.cpp")
EXAMPLE = os.path.join(ROOT, "examples", "depth_image_cloud.cpp")


@pytest.mark.parametrize("path", [SHIM, EXAMPLE])
def test_programs_compile(path):
    for flags in (["-Wall", "-Werror"], ["-Wall", "-Werror", *cxx.eigen_flags()]):
        r = cxx.syntax(path, flags=flags)
        assert r.returncode == 0, r.stderr


@pytest.mark.parametrize("decl", [
    "cilantro::DepthValueConverter<unsigned short, double> c(1000.0);",
    "cilantro::TruncatedDepthValueConverter<float, double> c(1000.0, 3.0);",
])
def test_double_metric_depth_is_a_compile_time_error(decl):
    src = f"#include <cilantro/core/image_point_cloud_conversions.hpp>\nvoid f() {{\n  {decl}\n}}\n"
    r = cxx.syntax(src=src)
    assert r.returncode != 0 and "float MetricDepth only" in r.stderr, r.stderr


def test_double_index_map_is_a_compile_time_error():
    src = ("#include <cilantro/core/image_point_cloud_conversions.hpp>\n"
           "void f(const cilantro::VectorSet3f& p, size_t* m) {\n"
           "  cilantro::pointsToIndexMap<double>(p, cilantro::b200::Intrinsics3f(), m, 4, 4);\n}\n")
    r = cxx.syntax(src=src)
    assert r.returncode != 0 and "float pointsToIndexMap only" in r.stderr, r.stderr


def test_existing_point_cloud_constructors_stay_unambiguous():
    src = ("#include <cilantro/utilities/point_cloud.hpp>\n#include <string>\n#include <vector>\n"
           "void f(const cilantro::PointCloud3f& c, const std::vector<size_t>& i, const std::vector<int>& j) {\n"
           "  cilantro::PointCloud3f a;\n  cilantro::PointCloud3f b(std::string(\"x.ply\"));\n"
           "  cilantro::PointCloud3f d(c, i);\n  cilantro::PointCloud3f e(c, j, true);\n  cilantro::PointCloud3f g(c);\n"
           "  (void)a; (void)b; (void)d; (void)e; (void)g;\n}\n")
    r = cxx.syntax(src=src, flags=("-Wall", "-Werror"))
    assert r.returncode == 0, r.stderr


def _back_records(cb, ctx, depth, rgb, K, T, conv):
    """The C ABI's results in the order the shim program writes them."""
    recs = []
    for ext in (None, T):
        for keep in (False, True):
            for normals, colour in ((False, None), (True, None), (False, rgb), (True, rgb)):
                recs.append(cb.depth_image_to_points(ctx, depth, K, conv, rgb=colour, extrinsics=ext, normals=normals,
                                                     keep_invalid=keep))
    recs.append(cb.depth_image_to_points(ctx, depth, K, conv, normals=True))
    recs.append(cb.depth_image_to_points(ctx, depth, K, conv, rgb=rgb))
    return recs


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,truncated", [(np.uint16, False), (np.uint16, True), (np.float32, False),
                                             (np.float32, True)])
def test_shim_program_equals_capi(cb, ctx, tmp_path, dtype, truncated):
    w, h = 47, 29
    depth = ref.frame("holed", w, h, dtype, seed=3)
    rgb = ref.rgb_frame(w, h, seed=3)
    K, T = ref.K_GENERAL, ref.pose(2, angle=0.05, shift=0.05)
    pts = np.asarray(ref.depth_to_points(depth, K, 1000.0, None)[0], np.float32)
    cols = np.random.default_rng(0).uniform(-0.1, 1.1, pts.shape).astype(np.float32)
    scale, md = 1000.0, (1.62 if truncated else 0.0)
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        np.array([w, h, int(dtype == np.float32), int(truncated), pts.shape[0]], np.int64).tofile(f)
        np.array([scale, md], np.float32).tofile(f)
        K.astype(np.float32).tofile(f)
        T.astype(np.float32).tofile(f)
        depth.tofile(f)
        rgb.tofile(f)
        pts.tofile(f)
        cols.tofile(f)
    out = tmp_path / "out.bin"
    cxx.run(cxx.build(SHIM, str(tmp_path / "test_depth_images_shim")), inp, out)
    raw = memoryview(open(out, "rb").read())
    off = 0

    def take(dt, count):
        nonlocal off
        a = np.frombuffer(raw[off:off + count * np.dtype(dt).itemsize], dt)
        off += count * np.dtype(dt).itemsize
        return a

    conv = cb.DepthConverter(dtype, scale, md if truncated else None)
    for r in _back_records(cb, ctx, depth, rgb, K, T, conv):
        m = int(take(np.int64, 1)[0])
        assert m == r["count"]
        for key in ("points", "normals", "colors"):
            if r.get(key) is not None:
                assert np.array_equal(take(np.uint32, 3 * m), r[key].view(np.uint32).reshape(-1)), key
    for ext in (None, T):
        d = cb.points_to_depth_image(ctx, pts, K, w, h, conv, extrinsics=ext)
        d2, im = cb.points_to_depth_image(ctx, pts, K, w, h, conv, colors=cols, extrinsics=ext)
        imap = cb.points_to_index_map(ctx, pts, K, w, h, extrinsics=ext)
        assert np.array_equal(take(dtype, w * h), d.reshape(-1))
        assert np.array_equal(take(dtype, w * h), d2.reshape(-1))
        assert np.array_equal(take(np.uint8, 3 * w * h), im.reshape(-1))
        i32 = np.where(imap == np.iinfo(np.uint64).max, np.iinfo(np.uint32).max, imap).astype(np.uint32)
        assert np.array_equal(take(np.uint32, w * h), i32.reshape(-1))
        assert np.array_equal(take(np.uint64, w * h), imap.reshape(-1))
    assert off == len(raw)


@pytest.mark.gpu
def test_example_runs(cb, tmp_path):
    out = cxx.run(cxx.build(EXAMPLE, str(tmp_path / "depth_image_cloud")), timeout=600, cwd=tmp_path)
    err = float(out.split("Pose error |T * pose^-1 - I|_F:")[1].split()[0])
    assert err < 1e-2
    out = cxx.run(cxx.build(EXAMPLE, str(tmp_path / "depth_image_cloud")),
                  os.path.join(ROOT, "tests", "golden", "scan_excerpt.ply"), timeout=600, cwd=tmp_path)
    assert "Pose error" in out
