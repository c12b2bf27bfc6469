"""The C++ drop-in surface of the dense warp-field ICP (SimpleCombinedMetricDenseRigidWarpFieldICP3f at
include/cilantro/registration/icp_common_instances.hpp) compiles without Eigen, together with the example program;
the GPU runs of both are in tests/test_gpu_warp_field.py."""
import os

import cxx

ROOT = cxx.ROOT


def _syntax(src_path=None, src=None):
    return cxx.syntax(src_path, src, flags=("-Wall", "-Werror"))


def test_warp_field_shim_and_example_compile_without_eigen():
    for path in (os.path.join(ROOT, "tests", "cpp", "test_warp_field_shim.cpp"),
                 os.path.join(ROOT, "examples", "non_rigid_icp_cloud.cpp")):
        r = _syntax(path)
        assert r.returncode == 0, r.stderr


def test_reference_spelling_of_the_dense_recipe_compiles():
    # the calls of the reference's examples/non_rigid_icp.cpp (dense variant), spelled as there
    src = ("#include <cilantro/registration/icp_common_instances.hpp>\n"
           "#include <cilantro/core/kd_tree.hpp>\n"
           "int main() { cilantro::VectorSet3f p(3, 4), n(3, 4);\n"
           "  std::vector<cilantro::NeighborSet<float>> nn;\n"
           "  cilantro::KDTree3f<>(p).search(p, cilantro::KNNNeighborhoodSpecification<>(12), nn);\n"
           "  cilantro::SimpleCombinedMetricDenseRigidWarpFieldICP3f icp(p, n, p, nn);\n"
           "  icp.correspondenceSearchEngine().setMaxDistance(0.04f * 0.04f);\n"
           "  icp.regularizationWeightEvaluator().setSigma(0.015f);\n"
           "  icp.setMaxNumberOfIterations(15).setConvergenceTolerance(2.5e-3f);\n"
           "  icp.setMaxNumberOfGaussNewtonIterations(1).setGaussNewtonConvergenceTolerance(5e-4f);\n"
           "  icp.setMaxNumberOfConjugateGradientIterations(500).setConjugateGradientConvergenceTolerance(1e-5f);\n"
           "  icp.setPointToPointMetricWeight(0.1f).setPointToPlaneMetricWeight(1.0f).setStiffnessRegularizationWeight(200.0f);\n"
           "  icp.setHuberLossBoundary(1e-2f);\n"
           "  auto tf_est = icp.estimate().getTransform();\n"
           "  cilantro::VectorSet3f out; cilantro::transformPoints(tf_est, p, out);\n"
           "  return (int)icp.getNumberOfPerformedIterations() + (int)icp.hasConverged(); }\n")
    r = _syntax(src=src)
    assert r.returncode == 0, r.stderr
