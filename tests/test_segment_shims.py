"""The C++ drop-in surface of the connected-component extraction (include/cilantro/clustering/
connected_component_extraction.hpp) compiles without Eigen, together with the example program; the GPU run of both is
in tests/test_gpu_segment.py."""
import os

from cxx import ROOT, syntax


def test_segment_shim_compiles_without_eigen():
    r = syntax(os.path.join(ROOT, "tests", "cpp", "test_segment_shim.cpp"))
    assert r.returncode == 0, r.stderr


def test_evaluators_compile_from_the_reference_include_path():
    src = ("#include <cilantro/core/common_pair_evaluators.hpp>\n"
           "int main() { cilantro::VectorSet3f n(3, 2), c(3, 2);\n"
           "  cilantro::NormalsProximityEvaluator<float, 3> a(n, 0.1f); cilantro::ColorsProximityEvaluator<float> b(c, 0.1f);\n"
           "  cilantro::PointsNormalsColorsProximityEvaluator<float, 3> d(n, c, 1.f, 0.1f, 0.1f);\n"
           "  return cilantro::AlwaysTrueEvaluator<float>()(0, 1, 0.f) ? 0 : 1; }\n")
    r = syntax(src=src)
    assert r.returncode == 0, r.stderr


def test_segment_example_compiles():
    r = syntax(os.path.join(ROOT, "examples", "segment_cloud.cpp"))
    assert r.returncode == 0, r.stderr


def test_an_evaluator_without_a_device_mapping_is_a_compile_error():
    src = ("#include <cilantro/clustering/connected_component_extraction.hpp>\n"
           "struct MyEvaluator { bool operator()(size_t, size_t, float) const { return true; } };\n"
           "int main() { cilantro::VectorSet3f p(3, 4);\n"
           "  cilantro::ConnectedComponentExtraction3f<>(p).segment(cilantro::RadiusNeighborhoodSpecification<float>(1.f),"
           " MyEvaluator()); }\n")
    r = syntax(src=src, flags=())
    assert r.returncode != 0 and "segment_fill" in r.stderr
