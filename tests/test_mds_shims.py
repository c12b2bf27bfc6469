"""The C++ drop-in of multidimensional scaling (MultidimensionalScaling<float, D>, MultidimensionalScaling2f / 3f / Xf,
computeDistancePreservingSpectralEmbedding, estimateEmbeddingDimensionEigengap): the header and the example compile with
and without Eigen, the double aliases are compile-time errors, and on the GPU the shim program gives the C ABI's results
bit for bit and the example runs."""
import os

import numpy as np
import pytest

import cxx
import mds_ref as mr

ROOT = cxx.ROOT
SHIM = os.path.join(ROOT, "tests", "cpp", "test_mds_shim.cpp")
EXAMPLE = os.path.join(ROOT, "examples", "multidimensional_scaling_cloud.cpp")


@pytest.mark.parametrize("path", [SHIM, EXAMPLE])
def test_programs_compile(path):
    for flags in (["-Wall", "-Werror"], ["-Wall", "-Werror", *cxx.eigen_flags()]):
        r = cxx.syntax(path, flags=flags)
        assert r.returncode == 0, r.stderr


@pytest.mark.parametrize("decl", [
    "cilantro::MultidimensionalScaling2d m(d);",
    "cilantro::MultidimensionalScaling3d m(d);",
    "cilantro::MultidimensionalScalingXd m(d, 2);",
    "cilantro::MultidimensionalScaling<double, 4> m(d);",
])
def test_double_instances_are_compile_time_errors(decl):
    src = ("#include <cilantro/utilities/multidimensional_scaling.hpp>\n"
           "struct M { const float* data() const { return nullptr; } size_t rows() const { return 0; }\n"
           "           size_t cols() const { return 0; } };\n"
           f"void f(const M& d) {{\n  {decl}\n}}\n")
    r = cxx.syntax(src=src)
    assert r.returncode != 0 and "float MultidimensionalScaling only" in r.stderr, r.stderr


def test_product_kernel_has_no_spills(tmp_path):
    """The symmetric product kernel (every block width and squaring variant) compiles for sm_90a without spills."""
    import subprocess

    from cilantro_b200 import build as cb_build

    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    src = os.path.join(ROOT, "cilantro_b200", "csrc", "mds.cu")
    r = subprocess.run([nvcc, *cb_build.NVCC_FLAGS, "-Xptxas", "-v", "-ccbin", "g++", "-c", "-o",
                        str(tmp_path / "mds.o"), src], capture_output=True, text=True, env=cxx.env())
    assert r.returncode == 0, r.stderr
    lines = r.stderr.splitlines()
    seen = 0
    for i, line in enumerate(lines):
        if "Function properties for" in line and "mds_product_kernel" in line:
            seen += 1
            assert "0 bytes spill stores, 0 bytes spill loads" in lines[i + 1], lines[i + 1]
    assert seen == 4


def _same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


@pytest.mark.gpu
@pytest.mark.parametrize("n,max_dim,est,squared,symmetric", [
    (300, 2, False, True, True), (300, 3, False, False, True), (257, 3, True, True, True), (40, 0, False, True, True),
    (120, 2, False, True, False)])
def test_shim_program_equals_capi(cb, ctx, tmp_path, n, max_dim, est, squared, symmetric):
    rng = np.random.default_rng(n + max_dim)
    p = rng.standard_normal((n, 4)) * np.array([3.0, 2.0, 1.0, 0.5])
    dm = mr.points_distances(p, squared=squared)
    if not symmetric:
        dm = (dm + rng.uniform(0, 0.3, dm.shape)).astype(np.float32)
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        np.array([n, max_dim, int(est), int(squared)], np.int64).tofile(f)
        np.asfortranarray(dm).T.copy().tofile(f)  # column-major: the transpose's rows
    out = tmp_path / "out.bin"
    exe = cxx.build(SHIM, str(tmp_path / "test_mds_shim"))
    cxx.run(exe, inp, out)
    raw = open(out, "rb").read()
    nev, dim, gap_dim = np.frombuffer(raw[:24], np.int64)
    vals = np.frombuffer(raw[24:], np.float32)
    xf_dim, xf_est = mr.xf_args(n, max_dim, est)
    want = cb.mds(ctx, dm, xf_dim, estimate_dim=xf_est, squared=squared)
    assert (nev, dim) == (want["eigenvalues"].size, want["dim"])
    assert gap_dim == mr.eigengap_dim(want["eigenvalues"], max_dim)
    off = 0

    def take(size):
        nonlocal off
        a = vals[off:off + size]
        off += size
        return a

    assert _same(take(nev), want["eigenvalues"])
    assert _same(take(n * dim), want["embedding"].reshape(-1))  # dim x n column-major = n x dim rows
    free = cb.mds(ctx, dm, max_dim, estimate_dim=est, squared=squared) if max_dim else None
    if free is not None:
        assert _same(take(free["eigenvalues"].size), free["eigenvalues"])
        assert _same(take(n * free["dim"]), free["embedding"].reshape(-1))
    if not est and max_dim in (2, 3):
        assert _same(take(nev), want["eigenvalues"]) and _same(take(n * dim), want["embedding"].reshape(-1))
    assert off == vals.size


@pytest.mark.gpu
def test_example_runs(cb, tmp_path):
    out = cxx.run(cxx.build(EXAMPLE, str(tmp_path / "multidimensional_scaling_cloud")), timeout=600, cwd=tmp_path)
    assert "Embedding dimension: 2" in out and "Stress:" in out
    stress = float(out.split("Stress:")[1].split()[0])
    assert 0.0 <= stress < 0.1
