"""The C++ drop-ins of the projective warp-field ICPs (SimpleCombinedMetricDenseRigidWarpFieldProjectiveICP3f and
SimpleCombinedMetricSparseRigidWarpFieldProjectiveICP3f in include/cilantro/correspondence_search/
correspondence_search_projective.hpp): the shim program and the example compile against the Eigen stub and against real
Eigen where present; the double and affine instances of the reference are not provided; on the GPU the example's call
sequence gives the C ABI's transforms, dense fields and correspondence lists bit for bit, a projection setter
re-attaches at the next estimate(), and the example tracks its frames."""
import os
import struct

import numpy as np
import pytest

import cxx

ROOT = cxx.ROOT
SHIM = os.path.join(ROOT, "tests", "cpp", "test_projective_warp_field_shim.cpp")
EXAMPLE = os.path.join(ROOT, "examples", "non_rigid_projective_tracking_cloud.cpp")
F = np.float32


def test_shim_and_example_compile_with_and_without_eigen():
    for flags in (["-Wall"], ["-Wall", *cxx.eigen_flags()]):
        for path in (SHIM, EXAMPLE):
            r = cxx.syntax(path, flags=flags)
            assert r.returncode == 0, r.stderr


@pytest.mark.parametrize("name", ["SimpleCombinedMetricDenseRigidWarpFieldProjectiveICP3d",
                                  "SimpleCombinedMetricSparseRigidWarpFieldProjectiveICP3d",
                                  "SimpleCombinedMetricDenseAffineWarpFieldProjectiveICP3f",
                                  "SimpleCombinedMetricSparseAffineWarpFieldProjectiveICP3f"])
def test_double_and_affine_instances_do_not_compile(name):
    src = ("#include <cilantro/registration/icp_common_instances.hpp>\n"
           f"int main() {{ return (int)sizeof(cilantro::{name}); }}\n")
    r = cxx.syntax(src=src, flags=())
    assert r.returncode != 0 and name in r.stderr, r.stderr


def read_runs(path):
    blob = open(path, "rb").read()
    runs, o = [], 0
    while o < len(blob):
        it, m, n, c = struct.unpack_from("<4Q", blob, o)
        o += 32
        T = np.frombuffer(blob, F, 12 * m, o).reshape(m, 3, 4)
        o += 48 * m
        Td = np.frombuffer(blob, F, 12 * n, o).reshape(n, 3, 4)
        o += 48 * n
        rec = np.frombuffer(blob, np.dtype([("a", "<u8"), ("b", "<u8"), ("v", "<f4")]), c, o)
        o += 20 * c
        runs.append(dict(iterations=it, T=T, T_dense=Td, first=rec["a"].astype(np.int64),
                         second=rec["b"].astype(np.int64), value=rec["v"].copy()))
    return runs


def same(got, want_T, want_list):
    assert np.array_equal(got["T"].view(np.uint32), np.asarray(want_T, F).view(np.uint32))
    f, s, v = want_list
    assert np.array_equal(got["first"], f) and np.array_equal(got["second"], s)
    assert np.array_equal(got["value"].view(np.uint32), v.view(np.uint32))


@pytest.mark.gpu
def test_shim_matches_capi(orc, tmp_path):
    import sparse_warp_field_ref as sref
    from cilantro_b200 import capi
    from test_gpu_projective_warp_field import lift

    P = lift(sref.make_case(6000, 0.025, seed=12), np.hstack([np.eye(3), np.zeros((3, 1))]).astype(F))
    (coff, cidx, cval), (roff, ridx, rval) = P["ctrl"], P["reg"]
    hdr = struct.pack("<8Q", P["dst"].shape[0], P["src"].shape[0], P["m"], cidx.shape[0], roff.shape[0] - 1,
                      ridx.shape[0], P["w"], P["h"])
    arrs = [np.asarray(P["K"], F), P["dst"], P["dst_normals"], P["src"], np.asarray(coff, np.uint64),
            np.asarray(cidx, np.int64), np.asarray(cval, F), np.asarray(roff, np.uint64), np.asarray(ridx, np.int64),
            np.asarray(rval, F)]
    scene = tmp_path / "scene.bin"
    scene.write_bytes(hdr + b"".join(np.ascontiguousarray(a).tobytes() for a in arrs))
    out = tmp_path / "runs.bin"
    cxx.run(cxx.build(SHIM, str(tmp_path / "shim")), scene, out, timeout=600)
    runs = read_runs(out)
    assert len(runs) == 3

    ctx = capi.Context(0)
    try:
        f32 = lambda a, b: float(F(a) * F(b))  # noqa: E731 (the C++ program's float products)
        kw = dict(w_pt=0.0, w_pl=1.0, stiffness=200.0, huber=1e-2, max_gn_iter=1, gn_tol=5e-4, max_cg_iter=500,
                  cg_tol=1e-5, reg_sigma=f32(3.0, 0.025), ctrl_sigma=f32(0.5, 0.025), max_iter=15, tol=2.5e-3,
                  max_d2=f32(0.02, 0.02))
        dst, src = capi.Cloud(ctx, P["dst"], P["dst_normals"]), capi.Cloud(ctx, P["src"])
        icp = capi.SparseWarpIcp(ctx, dst, src, P["ctrl"], P["m"], P["reg"])
        for run, w in zip(runs[:2], (P["w"], P["w"] - 8)):
            icp.set_projection(P["K"], w, P["h"])
            r = icp.estimate(**kw)
            same(run, r["T"], icp.correspondences())
            assert np.array_equal(run["T_dense"].view(np.uint32), r["T_dense"].view(np.uint32))
            assert run["iterations"] == r["iterations"] > 1 and run["first"].size == r["num_corr"] > 1000
        assert not np.array_equal(runs[0]["T"], runs[1]["T"])  # the narrower image re-attached
        nb = (np.zeros(1, np.uint64), np.zeros(0, np.int64), np.zeros(0, F))
        dense = capi.WarpIcp(ctx, dst, src, *nb)
        dense.set_projection(P["K"], P["w"], P["h"])
        r = dense.estimate(w_pt=0.1, w_pl=1.0, stiffness=200.0, max_gn_iter=1, max_cg_iter=500, max_iter=3,
                           max_d2=f32(0.04, 0.04))
        same(runs[2], r["T"], dense.correspondences())
        assert runs[2]["iterations"] == r["iterations"]
    finally:
        ctx.close()


@pytest.mark.gpu
def test_example_runs(tmp_path):
    out = cxx.run(cxx.build(EXAMPLE, str(tmp_path / "non_rigid_projective_tracking_cloud")), timeout=900,
                  cwd=tmp_path)
    assert "worst residual ratio" in out
