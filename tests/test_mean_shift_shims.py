"""The C++ drop-in surface of mean-shift (include/cilantro/clustering/mean_shift.hpp) compiles without Eigen, together
with the example program; the GPU runs of both are in tests/test_gpu_mean_shift.py."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = os.path.join(ROOT, "include")


def _env():
    env = dict(os.environ)
    env.pop("CXX", None)
    env.pop("CC", None)
    return env


def _syntax(src_path=None, src=None):
    cmd = ["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-I", INC]
    if src is None:
        return subprocess.run(cmd + [src_path], capture_output=True, text=True, env=_env())
    return subprocess.run(cmd + ["-x", "c++", "-"], input=src, capture_output=True, text=True, env=_env())


def test_mean_shift_shim_and_example_compile_without_eigen():
    for path in (os.path.join(ROOT, "tests", "cpp", "test_mean_shift_shim.cpp"),
                 os.path.join(ROOT, "examples", "mean_shift_cloud.cpp")):
        r = _syntax(path)
        assert r.returncode == 0, r.stderr


def test_weight_evaluators_take_the_reference_point_call():
    # mean_shift.hpp:64-66 calls evaluator(seed, point, d2)
    src = ("#include <cilantro/core/common_pair_evaluators.hpp>\n"
           "int main() { cilantro::Vector3f a(0.f, 0.f, 0.f), b(1.f, 0.f, 0.f);\n"
           "  float u = cilantro::UnityWeightEvaluator<float, float>()(a, b, 1.f);\n"
           "  float r = cilantro::RBFKernelWeightEvaluator<float, float, true>(1.f)(a, b, 1.f);\n"
           "  return (u == 1.f && r < 1.f) ? 0 : 1; }\n")
    r = _syntax(src=src)
    assert r.returncode == 0, r.stderr


def test_an_evaluator_without_a_device_mapping_is_a_compile_error():
    src = ("#include <cilantro/clustering/mean_shift.hpp>\n"
           "struct MyKernel { float operator()(size_t, size_t, float) const { return 1.f; } };\n"
           "int main() { cilantro::VectorSet3f p(3, 4);\n"
           "  cilantro::MeanShift3f<>(p).cluster(1.f, 10, 0.1f, 1e-6f, MyKernel()); }\n")
    r = _syntax(src=src)
    assert r.returncode != 0 and "b200_kind" in r.stderr
    src = ("#include <cilantro/clustering/mean_shift.hpp>\n"
           "int main() { cilantro::VectorSet3f p(3, 4);\n"
           "  cilantro::MeanShift3f<>(p).cluster(1.f, 10, 0.1f, 1e-6f, cilantro::RBFKernelWeightEvaluator<float, float, false>()); }\n")
    assert _syntax(src=src).returncode != 0
