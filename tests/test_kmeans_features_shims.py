"""The C++ drop-ins for k-means (KMeans<float, D>, KMeans2f<>, KMeans3f<>, KMeansXf<>, VectorSet<float, D>,
ConstVectorSetMatrixMap<float, D>): they compile without Eigen and with the Eigen stub (or a real Eigen), the
combinations the device path does not cover stay compile-time errors, and on the GPU the shim program gives the C ABI's
results bit for bit, clusters empty sets, and the coloured k-means example runs."""
import os

import numpy as np
import pytest

import cxx
import kmeans_ransac_ref as kr

ROOT = cxx.ROOT
SHIM = os.path.join(ROOT, "tests", "cpp", "test_kmeans_features_shim.cpp")
EIGEN = os.path.join(ROOT, "tests", "cpp", "test_kmeans_features_eigen.cpp")
EXAMPLE = os.path.join(ROOT, "examples", "colored_kmeans_cloud.cpp")


@pytest.mark.parametrize("path", [SHIM, EXAMPLE])
def test_programs_compile_without_eigen(path):
    r = cxx.syntax(path)
    assert r.returncode == 0, r.stderr


def test_containers_and_eigen_adapters(tmp_path):
    exe = cxx.build(EIGEN, str(tmp_path / "kmeans_features_eigen"), ["-Wall", "-I", cxx.INC, *cxx.eigen_flags()], link=False)
    cxx.run(exe)
    exe = cxx.build(EIGEN, str(tmp_path / "kmeans_features_no_eigen"), ["-Wall", "-I", cxx.INC, "-DCILANTRO_B200_NO_EIGEN"], link=False)
    cxx.run(exe)


@pytest.mark.parametrize("decl,message", [
    ("cilantro::KMeans<float, 3, cilantro::KDTreeDistanceAdaptors::L1> km(m3);", "L2 / L2Simple adaptors only"),
    ("cilantro::KMeans<float, 6, cilantro::KDTreeDistanceAdaptors::SO3> km(m6);", "L2 / L2Simple adaptors only"),
    ("cilantro::KMeans<double, 6> km(m6);", "float"),
    ("cilantro::KDTree<float, 6> tree(m6);", "<float, 3> instances only"),
    ("cilantro::VectorSet<double, 6> s;", "float vector sets only"),
])
def test_unsupported_instances_are_compile_time_errors(decl, message):
    src = ("#include <cilantro/clustering/kmeans.hpp>\n#include <cilantro/core/kd_tree.hpp>\n"
           "void f(const cilantro::ConstVectorSetMatrixMap3f& m3, const cilantro::ConstVectorSetMatrixMap<float, 6>& m6) {\n"
           f"  {decl}\n  (void)m3; (void)m6;\n}}\n")
    r = cxx.syntax(src=src)
    assert r.returncode != 0 and message in r.stderr, r.stderr


def _case(D, seed):
    rng = np.random.default_rng(seed)
    pts = np.vstack([kr.dyadic(rng, (300, D), 0.25) + np.float32(c) for c in (1.0, -1.5, 0.5, -0.25)]).astype(np.float32)
    return pts, pts[[0, 300, 600, 900, 5, 305]].copy()


@pytest.mark.gpu
@pytest.mark.parametrize("D", [6, 2, 3, 5])
def test_shim_program_equals_capi(cb, ctx, tmp_path, D):
    pts, cent0 = _case(D, D)
    n, k, max_iter, seed, tol = len(pts), len(cent0), 20, 7, 1e-4
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        np.array([n, D, k, max_iter, seed], np.int64).tofile(f)
        np.array([tol], np.float32).tofile(f)
        pts.tofile(f)
        cent0.tofile(f)
    out = tmp_path / "out.bin"
    exe = cxx.build(SHIM, str(tmp_path / "test_kmeans_features_shim"))
    cxx.run(exe, inp, out)
    raw = np.fromfile(out, np.uint8)
    v = cb.Vectors(ctx, pts)
    seeded = pts[cb.kmeans_seed_indices(n, k, seed)]
    off = 0
    for c0 in (cent0, seeded):
        want = cb.kmeans_cluster(ctx, v, c0, max_iter=max_iter, tol=tol)
        it = int(raw[off:off + 8].view(np.int64)[0])
        cent = raw[off + 8:off + 8 + 4 * k * D].view(np.float32).reshape(k, D)
        labels = raw[off + 8 + 4 * k * D:off + 8 + 4 * k * D + 8 * n].view(np.int64)
        off += 8 + 4 * k * D + 8 * n
        assert it == want["iterations"]
        assert np.array_equal(cent.view(np.uint32), want["centroids"].view(np.uint32))
        assert np.array_equal(labels, want["labels"])
    assert off == len(raw)


@pytest.mark.gpu
def test_colored_kmeans_example_runs(cb, tmp_path):
    out = cxx.run(cxx.build(EXAMPLE, str(tmp_path / "colored_kmeans_cloud")), timeout=600, cwd=tmp_path)
    assert "colored k-means:" in out and "k = 250" in out
