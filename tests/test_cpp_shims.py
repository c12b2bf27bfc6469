"""The C++ drop-in surface (include/cilantro/*.hpp over the C ABI): compiles without Eigen on CPU;
on the GPU box the reference-example calls in tests/cpp/test_shims.cpp run end to end."""
import os

import pytest

import cxx

ROOT = cxx.ROOT
SRC = os.path.join(ROOT, "tests", "cpp", "test_shims.cpp")


def test_shim_headers_compile_without_eigen():
    r = cxx.syntax(SRC)
    assert r.returncode == 0, r.stderr


@pytest.mark.gpu
def test_reference_examples_through_cpp_shims(cb, tmp_path):
    out = cxx.run(cxx.build(SRC, str(tmp_path / "test_shims")))
    assert "all C++ shim checks passed" in out


def test_eigen_adapters_type_check(tmp_path):
    """The `#if __has_include(<Eigen/Dense>)` adapters (VectorSet / ConstVectorSetMatrixMap / RigidTransform <-> Eigen).
    Eigen3 is absent from this image: they are compiled against tests/cpp/eigen_stub (a minimal stand-in with Eigen's
    layout and accessor names), or against the real Eigen where one is installed; host-only, no device call."""
    exe = cxx.build(os.path.join(ROOT, "tests", "cpp", "test_eigen_adapters.cpp"),
                    str(tmp_path / "test_eigen_adapters"), ["-Wall", *cxx.eigen_flags()])
    cxx.run(exe)


def test_example_program_compiles():
    r = cxx.syntax(os.path.join(ROOT, "examples", "register_clouds.cpp"))
    assert r.returncode == 0, r.stderr


@pytest.mark.gpu
def test_example_program_registers_a_synthetic_pair(cb, tmp_path):
    exe = cxx.build(os.path.join(ROOT, "examples", "register_clouds.cpp"), str(tmp_path / "register_clouds"))
    out = cxx.run(exe, cwd=str(tmp_path))
    assert "wrote registered.ply" in out and os.path.exists(tmp_path / "registered.ply")
