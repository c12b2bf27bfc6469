"""The C++ drop-in surface of the feature-space ICP: the feature adaptors (PointFeaturesAdaptor3f ...
PointNormalColorFeaturesAdaptor3f), CorrespondenceSearchKDTree<SearchFeatureAdaptorT> and the engine-templated
CombinedMetricRigidTransformICP3f / PointToPointMetricRigidTransformICP3f. The reference example's call sequence compiles
against the Eigen stub and against real Eigen where present; on the GPU the shim gives capi's transforms bit for bit, the
PointFeaturesAdaptor3f engine gives SimpleCombinedMetricRigidICP3f's, the pre-assembled feature matrix gives what the
(points, colours, weight) form gives, and the example runs."""
import os
import subprocess

import numpy as np
import pytest

from cilantro_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = os.path.join(ROOT, "include")
LIBDIR = os.path.join(ROOT, "cilantro_b200")
SHIM = os.path.join(ROOT, "tests", "cpp", "test_feature_icp_shim.cpp")
EXAMPLE = os.path.join(ROOT, "examples", "colored_icp_cloud.cpp")


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


def test_adaptor_constructors_match_the_feature_kind(tmp_path):
    """A constructor the adaptor kind does not have (e.g. colours for PointNormalFeaturesAdaptor3f's 5-argument form) does
    not compile, like the reference's."""
    src = tmp_path / "bad.cpp"
    src.write_text("#include <cilantro/correspondence_search/common_transformable_feature_adaptors.hpp>\n"
                   "int main() {\n"
                   "  cilantro::VectorSet3f p(3, 4), n(3, 4), c(3, 4);\n"
                   "  cilantro::PointNormalFeaturesAdaptor3f f(p, n, c, 0.5f, 5.0f);\n"
                   "  return 0;\n"
                   "}\n")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", INC, str(src)], capture_output=True, text=True,
                       env=_env())
    assert r.returncode != 0


def _run_shim(tmp_path, s):
    path = tmp_path / "scene.bin"
    np.concatenate([s[k].reshape(-1) for k in ("dst", "dst_normals", "dst_colors", "src", "src_normals",
                                               "src_colors")]).astype(np.float32).tofile(path)
    exe = _build(SHIM, str(tmp_path / "shim"))
    out = subprocess.run([exe, str(path), str(s["dst"].shape[0]), str(s["src"].shape[0])], capture_output=True,
                         text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    runs = {}
    for line in out.stdout.strip().splitlines():
        w = line.split()
        runs[w[0]] = (np.array(w[1:13], np.uint64).astype(np.uint32).view(np.float32).reshape(3, 4), int(w[13]),
                      int(w[14]))
    return runs


@pytest.mark.gpu
def test_shim_matches_capi(cb, ctx, tmp_path):
    s = synth.textured_sheet_pair(5000, seed=4)
    runs = _run_shim(tmp_path, s)
    kw = dict(metric="combined", w_pt=0.1, w_pl=1.0, max_iter=10, tol=0.0, max_d2=0.05)
    icp = cb.Icp(ctx, cb.Cloud(ctx, s["dst"], s["dst_normals"]), cb.Cloud(ctx, s["src"]))
    icp.set_features("point_normal_color", dst_normals=s["dst_normals"], dst_colors=s["dst_colors"],
                     src_normals=s["src_normals"], src_colors=s["src_colors"], normal_weight=0.5, color_weight=5.0)
    want = icp.estimate(**kw)
    T, it, nc = runs["feat"]
    assert np.array_equal(T.view(np.uint32), want["T"].view(np.uint32))
    assert (it, nc) == (want["iterations"], want["num_corr"])
    # PointFeaturesAdaptor3f as the engine = SimpleCombinedMetricRigidICP3f, bit for bit
    assert np.array_equal(runs["point"][0].view(np.uint32), runs["simple"][0].view(np.uint32))
    assert runs["point"][1:] == runs["simple"][1:]
    # the pre-assembled feature matrix = the (points, colours, weight) constructor
    assert np.array_equal(runs["color_pre"][0].view(np.uint32), runs["color"][0].view(np.uint32))
    assert runs["color_pre"][1:] == runs["color"][1:]
    # and the colour features register the in-plane shift the point-only ICP misses
    assert np.linalg.norm(runs["feat"][0][:2, 3] - s["T_ref"][:2, 3]) < 2e-3
    assert np.linalg.norm(runs["simple"][0][:2, 3] - s["T_ref"][:2, 3]) > 1e-2


@pytest.mark.gpu
def test_example_runs(tmp_path):
    exe = _build(EXAMPLE, str(tmp_path / "colored_icp_cloud"))
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600, cwd=tmp_path)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "in-plane offset error" in out.stdout
