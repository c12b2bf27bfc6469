"""The C++ drop-in surface of robust normal estimation: NormalEstimation<float, 3, MinimumCovarianceDeterminant<float, 3>>
(include/cilantro/core/normal_estimation.hpp, core/covariance.hpp) and PointCloud3f::removeInvalidNormals. The
reference example's call sequence compiles against the Eigen stub and against real Eigen where present, the whole-set
MinimumCovarianceDeterminant::operator() is a compile-time error, and on the GPU the shim gives capi's normals and the
example runs."""
import os
import subprocess

import numpy as np
import pytest

from cilantro_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = os.path.join(ROOT, "include")
LIBDIR = os.path.join(ROOT, "cilantro_b200")
SHIM = os.path.join(ROOT, "tests", "cpp", "test_robust_normals_shim.cpp")
EXAMPLE = os.path.join(ROOT, "examples", "robust_normal_estimation_cloud.cpp")


def _env():
    env = dict(os.environ)
    env.pop("CXX", None)
    env.pop("CC", None)
    return env


def _have_real_eigen():
    return subprocess.run(["g++", "-std=c++17", "-E", "-x", "c++", "-"], input="#include <Eigen/Dense>\n", text=True,
                          capture_output=True, env=_env()).returncode == 0


def _build(src, exe):
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", INC, src, "-o", exe, "-L", LIBDIR, "-lcilantro_b200",
                           f"-Wl,-rpath,{LIBDIR}"], env=_env())
    return exe


def test_shim_and_example_compile_with_and_without_eigen():
    incs = [["-I", INC], ["-I", INC] + ([] if _have_real_eigen() else ["-I", os.path.join(ROOT, "tests", "cpp",
                                                                                           "eigen_stub")])]
    for inc in incs:
        for path in (SHIM, EXAMPLE):
            r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", *inc, path], capture_output=True,
                               text=True, env=_env())
            assert r.returncode == 0, r.stderr


def test_whole_set_mcd_is_a_compile_time_error(tmp_path):
    src = tmp_path / "whole_set.cpp"
    src.write_text("#include <cilantro/core/covariance.hpp>\n"
                   "int main() {\n"
                   "  cilantro::MinimumCovarianceDeterminant<float, 3> mcd;\n"
                   "  cilantro::VectorSet3f pts(3, 10), cov(3, 3);\n"
                   "  cilantro::Vector3f mean;\n"
                   "  return mcd(cilantro::ConstVectorSetMatrixMap3f(pts), mean, cov) ? 0 : 1;\n"
                   "}\n")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", INC, str(src)], capture_output=True, text=True,
                       env=_env())
    assert r.returncode != 0 and "available inside NormalEstimation only" in r.stderr, r.stderr


@pytest.mark.gpu
def test_shim_matches_capi(cb, ctx, tmp_path):
    pts, _ = synth.surface_cloud(6000, seed=4, noise=0.0005)
    rng = np.random.default_rng(4)
    off = rng.random(pts.shape[0]) < 0.2
    pts[off, 2] += rng.uniform(0.01, 0.03, off.sum()).astype(np.float32)
    path = tmp_path / "points.bin"
    pts.astype(np.float32).tofile(path)
    exe = _build(SHIM, str(tmp_path / "shim"))
    out = subprocess.run([exe, str(path), "77"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = dict(line.split(" ", 1) for line in out.stdout.strip().splitlines())
    vals = np.array(lines["normals"].split()[1:], np.uint64).astype(np.uint32).view(np.float32).reshape(-1, 3)
    want = cb.Cloud(ctx, pts).estimate_normals_mcd(k=12, view_point=[0, 0, 0], num_trials=2, num_refinements=1,
                                                  chi_square_threshold=6.25, seed=77)
    assert np.array_equal(vals.view(np.uint32), want["normals"].view(np.uint32))
    assert int(lines["kept"]) == int((want["status"] == 0).sum()) < pts.shape[0]


@pytest.mark.gpu
def test_example_runs(cb, tmp_path):
    exe = _build(EXAMPLE, str(tmp_path / "example"))
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    line = [s for s in out.stdout.splitlines() if "invalid normals" in s][0]
    total, invalid = int(line.split()[0]), int(line.split()[2])
    assert 0 < invalid < total
    print(out.stdout)
