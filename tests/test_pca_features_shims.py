"""The C++ drop-ins for covariance and PCA over D-dimensional rows (Covariance<float, D>, PrincipalComponentAnalysis<float,
D>, PrincipalComponentAnalysis2f / Xf): they compile, PrincipalComponentAnalysis<float, 3> is
PrincipalComponentAnalysis3f, the instances the device path does not cover stay compile-time errors, and on the GPU the
shim program gives the C ABI's results bit for bit and the PCA example runs."""
import os

import numpy as np
import pytest

import cxx

ROOT = cxx.ROOT
SHIM = os.path.join(ROOT, "tests", "cpp", "test_pca_features_shim.cpp")
EXAMPLE = os.path.join(ROOT, "examples", "pca_features_cloud.cpp")


@pytest.mark.parametrize("path", [SHIM, EXAMPLE])
def test_programs_compile(path):
    r = cxx.syntax(path)
    assert r.returncode == 0, r.stderr


@pytest.mark.parametrize("decl,message", [
    ("cilantro::PrincipalComponentAnalysis<float, 6> p(m6, false, cilantro::MinimumCovarianceDeterminant<float, 3>());",
     "MinimumCovarianceDeterminant cov_eval is not implemented"),
    ("cilantro::PrincipalComponentAnalysis<double, 6> p(m6);", "float PrincipalComponentAnalysis only"),
    ("cilantro::Covariance<double, 6> c;", "float Covariance only"),
])
def test_unsupported_instances_are_compile_time_errors(decl, message):
    src = ("#include <cilantro/core/principal_component_analysis.hpp>\n"
           "void f(const cilantro::ConstVectorSetMatrixMap<float, 6>& m6) {\n"
           f"  {decl}\n  (void)m6;\n}}\n")
    r = cxx.syntax(src=src)
    assert r.returncode != 0 and message in r.stderr, r.stderr


def _same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


@pytest.mark.gpu
@pytest.mark.parametrize("D,k", [(2, 1), (3, 2), (6, 3), (9, 9), (40, 5)])
def test_shim_program_equals_capi(cb, ctx, tmp_path, D, k):
    rng = np.random.default_rng(D)
    n = 5003
    rows = (rng.standard_normal((n, D)) * rng.uniform(0.5, 3, D) + rng.uniform(-50, 50, D)).astype(np.float32)
    subset = np.concatenate([rng.integers(0, n, 700), [4, 4]]).astype(np.int64)
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        np.array([n, D, k, len(subset)], np.int64).tofile(f)
        rows.tofile(f)
        subset.tofile(f)
    out = tmp_path / "out.bin"
    exe = cxx.build(SHIM, str(tmp_path / "test_pca_features_shim"))
    cxx.run(exe, inp, out)
    raw = np.fromfile(out, np.float32)
    off = 0

    def take(shape):  # column-major in the file
        nonlocal off
        size = int(np.prod(shape))
        a = raw[off:off + size].reshape(shape[::-1]).T
        off += size
        return a

    v = cb.Vectors(ctx, rows)
    for sub in (None, subset):
        want = cb.pca(ctx, v, subset=sub)
        for key, shape in (("mean", (D,)), ("cov", (D, D)), ("eigenvalues", (D,)), ("eigenvectors", (D, D))):
            assert _same(take(shape), want[key]), (key, sub is None)
    m, c, ok = cb.mean_cov(ctx, v)
    assert ok and _same(take((D,)), m) and _same(take((D, D)), c)
    r = cb.pca(ctx, v)
    proj = cb.pca_project(ctx, v, r["mean"], r["eigenvectors"], k)
    assert _same(take((k, n)), proj.T)
    rec = cb.pca_reconstruct(ctx, cb.Vectors(ctx, proj), r["mean"], r["eigenvectors"])
    assert _same(take((D, n)), rec.T)
    assert off == raw.size


@pytest.mark.gpu
def test_pca_features_example_runs(cb, tmp_path):
    out = cxx.run(cxx.build(EXAMPLE, str(tmp_path / "pca_features_cloud")), timeout=600, cwd=tmp_path)
    assert "PCA<float, 9>:" in out and "explained variance" in out
