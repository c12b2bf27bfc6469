"""CPU-side checks of the product library (no GPU, no compute kernels):
  * libcilantro_b200.so loads and exports every symbol include/cilantro_b200.h declares;
  * without a device the library refuses to create a context (no CPU fallback);
  * the host-only O(1) solves agree with the oracle's independent implementations.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest

from cilantro_b200 import synth
from conftest import frob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    with open(os.path.join(ROOT, "include", "cilantro_b200.h")) as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    names = re.findall(r"\b(cb_[a-z0-9_]+)\s*\(", text)
    return sorted(set(names))


def test_library_exports_every_declared_symbol(cb):
    lib = cb.lib()
    declared = _declared_symbols()
    assert len(declared) >= 35
    missing = [s for s in declared if not hasattr(lib, s)]
    assert not missing, f"declared in include/cilantro_b200.h but not exported: {missing}"
    assert sorted(cb.EXPORTED) == declared, "capi.EXPORTED is out of sync with the header"
    assert b"sm_90a" in lib.cb_version()


def test_integration_guide_names_every_entry_point():
    """INTEGRATION.md is the maintainer's binding guide: every declared entry point appears there, either against the
    reference method it replaces or in the table of entry points without a reference counterpart."""
    with open(os.path.join(ROOT, "INTEGRATION.md")) as f:
        guide = f.read()
    missing = [s for s in _declared_symbols() if s not in guide]
    assert not missing, f"not mentioned in INTEGRATION.md: {missing}"


def test_no_cpu_fallback_without_device(cb):
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present; covered by the gpu tests")
    with pytest.raises(cb.CbError) as e:
        cb.Context(0)
    assert "no CPU fallback" in str(e.value) or "CUDA" in str(e.value)


def test_missing_library_fails_loudly(cb, monkeypatch):
    monkeypatch.setattr(cb, "_lib", None)
    monkeypatch.setattr(cb, "LIB_PATH", "/nonexistent/libcilantro_b200.so")
    with pytest.raises(cb.CbError):
        cb.lib()


def _moments(dst, src):
    d, s = dst.astype(np.float64), src.astype(np.float64)
    out = np.zeros(16)
    out[0] = d.shape[0]
    out[1:4] = d.sum(0)
    out[4:7] = s.sum(0)
    out[7:] = (d.T @ s).reshape(-1)
    return out


def test_solve_kabsch_moments_matches_oracle(cb, orc):
    rng = np.random.default_rng(0)
    for trial in range(20):
        n = int(rng.integers(3, 4000))
        src = rng.random((n, 3), dtype=np.float32)
        T = synth.rigid_from_axis_angle(rng.normal(size=3), rng.uniform(-1, 1), rng.normal(size=3) * 0.3)
        dst = synth.apply(T, src) + (rng.normal(size=(n, 3)) * 1e-3).astype(np.float32)
        if trial % 5 == 0:
            dst = dst * np.float32([1, 1, -1])  # forces the reflection branch
        Tp, okp = cb.solve_kabsch_moments(_moments(dst, src))
        To, oko = orc.kabsch(dst, src, accum_double=True)
        assert okp == oko
        # the mirrored case is ill-conditioned (the fix flips the axis of the smallest singular value;
        # the oracle rounds sigma to fp32 like the reference, the product keeps double)
        assert frob(Tp, To) < (5e-5 if trial % 5 == 0 else 2e-6), (trial, frob(Tp, To))
        assert abs(np.linalg.det(Tp[:, :3].astype(np.float64)) - 1) < 1e-5
    # 3 points (RANSAC sample): rank-deficient covariance
    src = rng.random((3, 3), dtype=np.float32)
    dst = synth.apply(T, src)
    Tp, okp = cb.solve_kabsch_moments(_moments(dst, src))
    To, _ = orc.kabsch(dst, src, accum_double=True)
    assert okp and frob(Tp, To) < 5e-6
    assert np.abs(synth.apply(Tp, src) - dst).max() < 1e-5
    # no pairs -> identity, false (transform_estimation.hpp:20-23)
    Tp, okp = cb.solve_kabsch_moments(np.zeros(16))
    assert not okp and frob(Tp, orc.identity()) == 0


def test_solve_gauss_newton_matches_oracle(cb, orc):
    rng = np.random.default_rng(1)
    dst, src, nrm, T_ref = synth.icp_pair(3000, seed=8, noise=0.0005, with_normals=True)
    q = synth.apply(T_ref, src)  # almost aligned
    idx = np.arange(3000)
    for w_pt, w_pl in ((0.0, 1.0), (0.3, 1.0), (1.0, 0.0)):
        # build the normal equations exactly as the kernel does (double precision)
        d = dst.astype(np.float64)
        s = q.astype(np.float64)
        v, e = d + s, d - s
        A = np.zeros((6, 6))
        b = np.zeros(6)
        if w_pl > 0:
            a = np.hstack([np.cross(v, nrm.astype(np.float64)), nrm.astype(np.float64)])
            r = (nrm.astype(np.float64) * e).sum(1)
            A += w_pl * a.T @ a
            b += w_pl * a.T @ r
        if w_pt > 0:
            for i in range(3000):
                vx = np.array([[0, -v[i, 2], v[i, 1]], [v[i, 2], 0, -v[i, 0]], [-v[i, 1], v[i, 0], 0]])
                E = np.vstack([vx, np.eye(3)])  # eq_vecs, transform_estimation.hpp:306-316
                A += w_pt * E @ E.T
                b += w_pt * E @ e[i]
        sums = np.zeros(28)
        sums[0] = 3000
        sums[1:22] = A[np.triu_indices(6)]
        sums[22:] = b
        Tp, dn = cb.solve_gauss_newton(sums)
        To, _ = orc.estimate_combined(dst, nrm, q, idx, idx, w_pt, w_pl, 1, 1e-5, accum_double=True)
        assert frob(Tp, To) < 2e-6, (w_pt, w_pl, frob(Tp, To))
        assert dn > 0


def test_solve_rotation_and_compose(cb, orc):
    rng = np.random.default_rng(2)
    for _ in range(20):
        R = synth.rigid_from_axis_angle(rng.normal(size=3), rng.uniform(-3, 3), [0, 0, 0])[:, :3]
        noisy = (R + 1e-4 * rng.normal(size=(3, 3))).astype(np.float32)
        assert np.abs(cb.solve_rotation(noisy) - orc.rotation(noisy)).max() < 1e-6
    A = synth.rigid_from_axis_angle([1, 0, 0], 0.3, [1, 2, 3]).astype(np.float32)
    B = synth.rigid_from_axis_angle([0, 1, 0], -0.2, [-1, 0, 4]).astype(np.float32)
    AB = cb.compose(A, B)
    p = rng.random((10, 3), dtype=np.float32)
    assert np.abs(synth.apply(AB, p) - synth.apply(A, synth.apply(B, p))).max() < 1e-5


def test_kmeans_seed_indices_host(cb, orc):
    assert np.array_equal(cb.kmeans_seed_indices(5000, 100, 42), orc.kmeans_seed_indices(5000, 100, 42))


def test_product_never_touches_the_oracle():
    """The oracle is test infrastructure: nothing under cilantro_b200/ or include/ may include, import, link or
    dlopen it, and the shared library must not depend on it."""
    import re
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pat = re.compile(r'#\s*include\s*[<"][^>"\n]*oracle|^\s*import\s+oracle\b|^\s*from\s+oracle\b.*\bimport\b|'
                     r'libcilantro_oracle|libcilantro_ref_knn|\borc_[a-z_]+\s*\(', re.M)
    offenders = []
    for base in ("cilantro_b200", "include"):
        for dirpath, _, files in os.walk(os.path.join(root, base)):
            for f in files:
                if not f.endswith((".py", ".cu", ".cuh", ".hpp", ".h", ".cpp")):
                    continue
                text = open(os.path.join(dirpath, f), errors="ignore").read()
                if pat.search(text):
                    offenders.append(os.path.join(dirpath, f))
    assert not offenders, offenders
    lib = os.path.join(root, "cilantro_b200", "libcilantro_b200.so")
    needed = subprocess.run(["readelf", "-d", lib], capture_output=True, text=True).stdout
    assert "oracle" not in needed and "ref_knn" not in needed


def test_library_carries_only_sm_90a_code():
    """Built for H100 and nothing else: every embedded cubin is sm_90a (no multi-arch fat binary, no PTX-only JIT
    path), and the hot kernels are in it."""
    import shutil
    import subprocess

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    lib = os.path.join(ROOT, "cilantro_b200", "libcilantro_b200.so")
    elfs = [ln for ln in subprocess.run(["cuobjdump", "-lelf", lib], capture_output=True, text=True).stdout.splitlines()
            if ln.startswith("ELF file")]
    assert elfs and all(".sm_90a.cubin" in ln for ln in elfs), elfs
    syms = subprocess.run(["cuobjdump", "-symbols", lib], capture_output=True, text=True).stdout
    for kernel in ("icp_pass_kernel", "icp_search_kernel", "icp_cached_pipe_kernel", "icp_finish_kernel",
                   "kmeans_assign_kernel", "ransac_score_kernel", "moments_kernel", "normals_knn_kernel",
                   "radix_scatter_kernel", "bin_reduce_kernel", "pairs_pass_kernel"):
        assert kernel in syms, kernel
    # the asynchronous-copy pipeline of the cached pass and the programmatic dependent launch of the loop kernels made
    # it into the SASS (cp.async -> LDGSTS / LDGDEPBAR, griddepcontrol.wait / launch_dependents -> ACQBULK / PREEXIT)
    sass = subprocess.run(["cuobjdump", "-sass", "-fun", "icp_cached_pipe_kernel", lib], capture_output=True, text=True).stdout
    if "LDGSTS" not in sass:  # older cuobjdump: no demangled -fun match, fall back to the whole library
        sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
    for mnemonic in ("LDGSTS", "LDGDEPBAR", "ACQBULK", "PREEXIT"):
        assert mnemonic in sass, mnemonic


def _kabsch_numpy(d, q):
    """estimateTransformPointToPointMetric (transform_estimation.hpp:12-48) with numpy: R = U V^T of
    sigma = (d - mu_d)(q - mu_q)^T / n, reflection fixed on the LAST column of U."""
    mud, muq = d.mean(0), q.mean(0)
    sigma = (d - mud).T @ (q - muq) / len(d)
    U, S, Vt = np.linalg.svd(sigma)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        U[:, 2] = -U[:, 2]
    R = U @ Vt
    return np.hstack([R, (mud - R @ muq)[:, None]])


@pytest.mark.parametrize("case", ["generic", "near_identity", "planar", "reflection", "collinear"])
def test_rotation_solver_polar_and_svd_paths(cb, case):
    """solve_core.hpp takes the polar (Newton) iteration when det > 0 and the matrix is well conditioned, and the
    Jacobi SVD otherwise (reflection / rank-deficient rules): both against numpy's SVD, on inputs built to hit each."""
    rng = np.random.default_rng({"generic": 1, "near_identity": 2, "planar": 3, "reflection": 4, "collinear": 5}[case])
    worst = 0.0
    for _ in range(50):
        n = 60
        q = rng.normal(size=(n, 3))
        if case == "planar":
            q[:, 2] = 0.0  # sigma has a zero singular value: SVD path, u2 = u0 x u1
        if case == "collinear":
            q[:, 1:] = 0.0
        ang = rng.normal(size=3) * (0.01 if case == "near_identity" else 1.0)
        th = np.linalg.norm(ang)
        k = ang / th
        K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
        R = np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * (K @ K)
        d = q @ R.T + rng.normal(size=3)
        if case == "reflection":
            d = d * np.array([1.0, 1.0, -1.0]) + 1e-3 * rng.normal(size=(n, 3))  # det(sigma) < 0: Kabsch must still return a rotation
        s = np.zeros(16)
        s[0] = n
        s[1:4] = d.sum(0)
        s[4:7] = q.sum(0)
        s[7:16] = (d.T @ q).ravel()
        T, ok = cb.solve_kabsch_moments(s)
        assert ok
        Rg = T[:, :3].astype(np.float64)
        assert abs(np.linalg.det(Rg) - 1.0) < 1e-5 and np.abs(Rg @ Rg.T - np.eye(3)).max() < 1e-5
        if case in ("generic", "near_identity", "reflection"):
            worst = max(worst, np.abs(T - _kabsch_numpy(d, q)).max())
        else:  # rank-deficient: the rotation is not unique, but it must map the points correctly
            worst = max(worst, np.abs((q @ Rg.T + T[:, 3]) - d).max())
    assert worst < 2e-5, worst


def test_icp_params_layout_matches_the_header(cb):
    """capi.IcpParams mirrors struct cb_icp_params field by field (order and count; sizes follow from the types)."""
    hdr = open(os.path.join(ROOT, "include", "cilantro_b200.h")).read()
    body = hdr[hdr.index("typedef struct cb_icp_params {"):hdr.index("} cb_icp_params;")]
    names = re.findall(r"^\s*(?:int32_t|float|double)\s+(\w+)(?:\[\d+\])?;", body, re.M)
    assert names == [f[0] for f in cb.IcpParams._fields_], (names, [f[0] for f in cb.IcpParams._fields_])
    p = cb.icp_params(pt_rbf_sigma=0.5, host_loop=True)
    assert p.host_loop == 1 and p.pt_weight_kind == 1 and abs(p.pt_weight_coeff + 2.0) < 1e-6 and p.pl_weight_kind == 0
