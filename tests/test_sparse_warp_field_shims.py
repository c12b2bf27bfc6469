"""The C++ drop-in surface of the sparse warp-field ICP (SimpleCombinedMetricSparseRigidWarpFieldICP3f at
include/cilantro/registration/icp_common_instances.hpp) compiles without Eigen, together with the example program and
the calls of the reference example's sparse recipe; the GPU runs are in tests/test_gpu_sparse_warp_field.py."""
import os

from test_warp_field_shims import ROOT, _syntax


def test_sparse_warp_field_shim_and_example_compile_without_eigen():
    for path in (os.path.join(ROOT, "tests", "cpp", "test_sparse_warp_field_shim.cpp"),
                 os.path.join(ROOT, "examples", "sparse_non_rigid_icp_cloud.cpp")):
        r = _syntax(path)
        assert r.returncode == 0, r.stderr


def test_reference_spelling_of_the_sparse_recipe_compiles():
    # the calls of the reference's examples/non_rigid_icp.cpp (sparse variant), spelled as there
    src = ("#include <cilantro/registration/icp_common_instances.hpp>\n"
           "#include <cilantro/utilities/point_cloud.hpp>\n"
           "int main() { cilantro::PointCloud3f dst, src;\n"
           "  float control_res = 0.025f;\n"
           "  cilantro::VectorSet<float, 3> control_points =\n"
           "      cilantro::PointsGridDownsampler3f(src.points, control_res).getDownsampledPoints();\n"
           "  cilantro::KDTree<float, 3> control_tree(control_points);\n"
           "  cilantro::NeighborhoodSet<float> src_to_control_nn =\n"
           "      control_tree.search(src.points, cilantro::KNNNeighborhoodSpecification<>(4));\n"
           "  cilantro::NeighborhoodSet<float> regularization_nn =\n"
           "      control_tree.search(control_points, cilantro::KNNNeighborhoodSpecification<>(8));\n"
           "  cilantro::SimpleCombinedMetricSparseRigidWarpFieldICP3f icp(\n"
           "      dst.points, dst.normals, src.points, src_to_control_nn, control_points.cols(), regularization_nn);\n"
           "  icp.correspondenceSearchEngine().setMaxDistance(0.02f * 0.02f);\n"
           "  icp.controlWeightEvaluator().setSigma(0.5f * control_res);\n"
           "  icp.regularizationWeightEvaluator().setSigma(3.0f * control_res);\n"
           "  icp.setMaxNumberOfIterations(15).setConvergenceTolerance(2.5e-3f);\n"
           "  icp.setMaxNumberOfGaussNewtonIterations(1).setGaussNewtonConvergenceTolerance(5e-4f);\n"
           "  icp.setMaxNumberOfConjugateGradientIterations(500).setConjugateGradientConvergenceTolerance(1e-5f);\n"
           "  icp.setPointToPointMetricWeight(0.0f).setPointToPlaneMetricWeight(1.0f).setStiffnessRegularizationWeight(200.0f);\n"
           "  icp.setHuberLossBoundary(1e-2f);\n"
           "  auto tf_est = icp.estimate().getDenseWarpField();\n"
           "  auto residuals = icp.getResiduals();\n"
           "  auto warped = src.transformed(tf_est);\n"
           "  return (int)icp.getNumberOfPerformedIterations() + (int)icp.hasConverged() + (int)residuals.size() +\n"
           "         (int)warped.size(); }\n")
    r = _syntax(src=src)
    assert r.returncode == 0, r.stderr
