"""ORACLE — test infrastructure, NOT product code: ctypes binding of the sparse warp-field restatement
(oracle/sparse_warp_field_oracle.cpp -> oracle/libsparse_warp_oracle.so, built on first use or by build()) and the
serial ICP loop of CombinedMetricSparseWarpFieldICP on the oracle's brute-force 1-NN.

    from oracle import sparse_warp_field
    sparse_warp_field.icp(dst, dst_n, src, ctrl, n_ctrl, reg, max_iter=5, w_pt=0.0, stiffness=200.0)

ctrl = (offsets, index, value): one control list of (node, squared distance) per source point; reg = the node
neighbourhoods' CSR. Node transforms are (n_ctrl, 3, 4) float32, dense transforms (n_src, 3, 4).
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import warp_field as _dense

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "sparse_warp_field_oracle.cpp")
_LIB_PATH = os.path.join(_HERE, "libsparse_warp_oracle.so")
_lib = None


def build(force=False):
    deps = [_SRC, os.path.join(_HERE, "warp_field_oracle.cpp"), os.path.join(_HERE, "small_linalg.hpp")]
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < max(os.path.getmtime(d) for d in deps):
        env = dict(os.environ)
        env.pop("CXX", None)
        tmp = _LIB_PATH + f".{os.getpid()}.tmp"
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fPIC", "-shared",
                               "-fvisibility=hidden", "-Wall", "-o", tmp, _SRC], env=env)
        os.replace(tmp, _LIB_PATH)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_sparse_warp_solve.restype = C.c_int
        _lib.orc_sparse_warp_system.restype = None
        _lib.orc_sparse_warp_resample.restype = None
    return _lib


_p = _dense._p
_f32 = _dense._f32
_nbhd = _dense._nbhd
rbf_coeff = _dense.rbf_coeff
apply = _dense.apply
compose = _dense.compose
residuals = _dense.residuals


def _ctrl_args(ctrl, n_ctrl, ctrl_sigma):
    off, idx, val = _nbhd(ctrl)
    return [_p(off), _p(idx), _p(val), C.c_size_t(int(n_ctrl)), C.c_float(rbf_coeff(ctrl_sigma))], (off, idx, val)


def resample(T_ctrl, ctrl, n_ctrl, ctrl_sigma=1.0):
    """resampleTransforms in the device's float order: (n_src, 3, 4) from the node transforms."""
    args, keep = _ctrl_args(ctrl, n_ctrl, ctrl_sigma)
    n = keep[0].shape[0] - 1
    T = np.ascontiguousarray(T_ctrl, np.float32).reshape(-1, 12)
    out = np.empty((max(n, 1), 12), np.float32)
    lib().orc_sparse_warp_resample(C.c_size_t(n), *args, _p(T), _p(out))
    return out[:n].reshape(n, 3, 4)


def system(dst, dst_n, src, first, second, ctrl, n_ctrl, reg, x, p, w_pt=0.0, w_pl=1.0, stiffness=1.0,
           huber_delta=1e-4, reg_sigma=1.0, ctrl_sigma=1.0):
    """The normal equations in double at the node unknowns x (m, 6): dict(b, diag, q = At At^T p), each (m, 6)."""
    dst, src = _f32(dst), _f32(src)
    dn = None if dst_n is None else _f32(dst_n)
    m = int(n_ctrl)
    cargs, _ = _ctrl_args(ctrl, n_ctrl, ctrl_sigma)
    roff, ridx, rval = _nbhd(reg)
    f = np.ascontiguousarray(first, np.uint64)
    s = np.ascontiguousarray(second, np.uint64)
    x = np.ascontiguousarray(x, np.float64).reshape(m, 6)
    pv = np.ascontiguousarray(p, np.float64).reshape(m, 6)
    b = np.empty((max(m, 1), 6)); diag = np.empty((max(m, 1), 6)); q = np.empty((max(m, 1), 6))
    lib().orc_sparse_warp_system(_p(dst), _p(dn), C.c_size_t(src.shape[0]), _p(src), *cargs, C.c_size_t(f.shape[0]),
                                 _p(f), _p(s), _p(roff), _p(ridx), _p(rval), C.c_size_t(max(roff.shape[0] - 1, 0)),
                                 C.c_float(w_pt), C.c_float(w_pl), C.c_float(stiffness), C.c_float(huber_delta),
                                 C.c_float(rbf_coeff(reg_sigma)), _p(x), _p(pv), _p(b), _p(diag), _p(q))
    return {"b": b[:m], "diag": diag[:m], "q": q[:m]}


def solve(dst, dst_n, src, first, second, ctrl, n_ctrl, reg, w_pt=0.0, w_pl=1.0, stiffness=1.0, huber_delta=1e-4,
          reg_sigma=1.0, ctrl_sigma=1.0, max_gn_iter=10, gn_tol=1e-5, max_cg_iter=1000, cg_tol=1e-5, double=False):
    """estimateSparseWarpFieldCombinedMetric on src (already warped). Returns dict(T (m, 3, 4), x (m, 6), converged,
    gn_steps, cg_iterations, cg_iterations_last, cg_error)."""
    dst, src = _f32(dst), _f32(src)
    dn = None if dst_n is None else _f32(dst_n)
    m = int(n_ctrl)
    cargs, _ = _ctrl_args(ctrl, n_ctrl, ctrl_sigma)
    roff, ridx, rval = _nbhd(reg)
    f = np.ascontiguousarray(first, np.uint64)
    s = np.ascontiguousarray(second, np.uint64)
    T = np.empty((max(m, 1), 12), np.float32)
    x = np.empty((max(m, 1), 6), np.float32)
    st = np.zeros(4, np.uint64)
    err = C.c_float()
    lib().orc_sparse_warp_solve(C.c_size_t(dst.shape[0]), _p(dst), _p(dn), C.c_size_t(src.shape[0]), _p(src), *cargs,
                                C.c_size_t(f.shape[0]), _p(f), _p(s), _p(roff), _p(ridx), _p(rval),
                                C.c_size_t(max(roff.shape[0] - 1, 0)), C.c_float(w_pt), C.c_float(w_pl),
                                C.c_float(stiffness), C.c_float(huber_delta), C.c_float(rbf_coeff(reg_sigma)),
                                C.c_uint64(int(max_gn_iter)), C.c_float(gn_tol), C.c_uint64(int(max_cg_iter)),
                                C.c_float(cg_tol), C.c_int(int(double)), _p(T), _p(x), _p(st), C.byref(err))
    return {"T": T[:m].reshape(m, 3, 4), "x": x[:m], "converged": bool(st[0]), "gn_steps": int(st[1]),
            "cg_iterations": int(st[2]), "cg_iterations_last": int(st[3]), "cg_error": float(err.value)}


def icp(dst, dst_n, src, ctrl, n_ctrl, reg, knn=None, T_init=None, max_iter=15, tol=1e-5, max_d2=1e-4, double=False,
        ctrl_sigma=1.0, **kw):
    """CombinedMetricSparseWarpFieldICP::estimate() (icp_base.hpp:68-87): the dense field resampled from the nodes,
    then per iteration the 1-NN of T_i s_i within max_d2, the estimator (solve(), kw = its parameters), the nodes'
    T_j <- rotation(dT_j T_j) and the resampling again. Returns dict(T, T_dense, iterations, converged, last_delta,
    num_corr, gn_steps, cg_iterations, first, second)."""
    import oracle

    dst, src = _f32(dst), _f32(src)
    knn = knn or oracle.BruteKnn(dst)
    n, m = src.shape[0], int(n_ctrl)
    T = np.tile(np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32), (m, 1, 1)) if T_init is None else \
        np.array(T_init, np.float32).reshape(m, 3, 4)
    T = np.ascontiguousarray(T)
    Td = resample(T, ctrl, m, ctrl_sigma)
    it, last, steps, cgi = 0, float("inf"), 0, 0
    first = second = np.zeros(0, np.int64)
    while it < max_iter:
        q = apply(Td, src)
        idx, _ = knn.query(q, max_d2) if dst.shape[0] else (np.full(n, -1), None)
        second = np.nonzero(idx >= 0)[0]
        first = idx[second]
        r = solve(dst, dst_n, q, first, second, ctrl, m, reg, double=double, ctrl_sigma=ctrl_sigma, **kw)
        steps += r["gn_steps"]
        cgi += r["cg_iterations"]
        last = float(np.sqrt(np.float32(compose(r["T"].reshape(m, 12), T.reshape(m, 12))))) if m else 0.0
        Td = resample(T, ctrl, m, ctrl_sigma)
        it += 1
        if last < tol:
            break
    return {"T": T, "T_dense": Td, "iterations": it, "converged": it > 0 and last < tol, "last_delta": last,
            "num_corr": int(second.shape[0]), "gn_steps": steps, "cg_iterations": cgi, "first": first,
            "second": second}
