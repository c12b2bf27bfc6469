"""The C++ drop-in surface of projective ICP (include/cilantro/correspondence_search/correspondence_search_projective.hpp):
CorrespondenceSearchProjective<float>, SimpleCombinedMetricRigidProjectiveICP3f and the engine-templated ICPs over it.
The shim program and the example compile against the Eigen stub and against real Eigen where present; every other
ScalarT, evaluation adaptor or evaluator is a compile-time error; on the GPU the fusion example's call sequence gives
capi's transforms, iteration counts and correspondence counts bit for bit, a projection setter re-attaches at the next
estimate(), and the example tracks its trajectory."""
import os
import struct

import numpy as np
import pytest

import cxx
import depth_images_ref as dimg
import icp_ref

ROOT = cxx.ROOT
SHIM = os.path.join(ROOT, "tests", "cpp", "test_projective_icp_shim.cpp")
EXAMPLE = os.path.join(ROOT, "examples", "projective_tracking_cloud.cpp")
F = np.float32


def test_shim_and_example_compile_with_and_without_eigen():
    for flags in (["-Wall"], ["-Wall", *cxx.eigen_flags()]):
        for path in (SHIM, EXAMPLE):
            r = cxx.syntax(path, flags=flags)
            assert r.returncode == 0, r.stderr


@pytest.mark.parametrize("args, what", [
    ("double", "float projective search only"),
    ("float, cilantro::PointNormalFeaturesAdaptor3f", "PointFeaturesAdaptor3f only"),
    ("float, cilantro::PointFeaturesAdaptor3f, cilantro::RBFKernelWeightEvaluator<float, float>", "DistanceEvaluator"),
])
def test_other_instances_do_not_compile(args, what):
    src = ("#include <cilantro/correspondence_search/correspondence_search_projective.hpp>\n"
           f"int main() {{ return (int)sizeof(cilantro::CorrespondenceSearchProjective<{args}>); }}\n")
    r = cxx.syntax(src=src, flags=())
    assert r.returncode != 0 and what in r.stderr, r.stderr


def scene(w=160, h=120):
    f = F(0.8 * w)
    K = np.array([[f, 0, (w - 1) / 2], [0, f, (h - 1) / 2], [0, 0, 1]], F)
    E = dimg.pose(3, 0.1, 0.05)
    depth = dimg.frame("full", w, h, np.float32, seed=21)
    dst, dst_n, _ = dimg.depth_to_points(depth, K, 1000.0, None, None, E, normals=True)
    T = dimg.pose(22, 0.02, 0.01)
    Ti = np.hstack([T[:, :3].T, -(T[:, :3].T @ T[:, 3:].astype(np.float64))]).astype(F)
    src = icp_ref.apply_f32(Ti, dst)
    src_n = (dst_n.astype(np.float64) @ T[:, :3].astype(np.float64)).astype(F)
    return dict(K=K, E=E, w=w, h=h, T0=icp_ref.identity().astype(F), dst=dst, dst_n=dst_n, src=src, src_n=src_n)


def run_shim(tmp_path, s):
    path = tmp_path / "scene.bin"
    blob = struct.pack("<QQQQ", s["dst"].shape[0], s["src"].shape[0], s["w"], s["h"])
    blob += b"".join(np.asarray(s[k], F).tobytes() for k in ("K", "E", "T0", "dst", "dst_n", "src", "src_n"))
    path.write_bytes(blob)
    out = cxx.run(cxx.build(SHIM, str(tmp_path / "shim")), path)
    runs = {}
    for line in out.strip().splitlines():
        w = line.split()
        if w[0] == "defaults":
            runs["defaults"] = int(w[1])
            continue
        runs[w[0]] = (np.array(w[1:13], np.uint64).astype(np.uint32).view(F).reshape(3, 4), int(w[13]), int(w[14]))
    return runs


@pytest.mark.gpu
def test_shim_matches_capi(cb, ctx, tmp_path):
    s = scene()
    runs = run_shim(tmp_path, s)
    assert runs["defaults"] == 1
    kw = dict(max_d2=F(0.1 * 0.1), T_init=s["T0"], tol=5e-4, max_iter=6)
    for name, metric, src_n in (("simple", "combined", None), ("symmetric", "combined", s["src_n"]),
                                ("p2p", "p2p", None)):
        icp = cb.Icp(ctx, cb.Cloud(ctx, s["dst"], s["dst_n"]), cb.Cloud(ctx, s["src"], src_n))
        icp.set_projection(s["K"], s["w"], s["h"], s["E"])
        extra = dict(w_pt=0.0, w_pl=1.0, max_opt_iter=1) if metric == "combined" else {}
        want = icp.estimate(metric=metric, **kw, **extra)
        T, it, nc = runs[name]
        assert np.array_equal(T.view(np.uint32), want["T"].view(np.uint32)), name
        assert (it, nc) == (want["iterations"], want["num_corr"]), name
        assert nc > 1000
    # an estimate() with nothing changed gives the same result; a setter re-attaches (an empty image: no pairs)
    assert np.array_equal(runs["again"][0].view(np.uint32), runs["simple"][0].view(np.uint32))
    assert runs["again"][1:] == runs["simple"][1:]
    assert runs["empty"][2] == 0


@pytest.mark.gpu
def test_example_runs(tmp_path):
    out = cxx.run(cxx.build(EXAMPLE, str(tmp_path / "projective_tracking_cloud")), timeout=600, cwd=tmp_path)
    assert "worst pose error" in out
