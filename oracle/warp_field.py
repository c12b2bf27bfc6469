"""ORACLE — test infrastructure, NOT product code: ctypes binding of the dense warp-field restatement
(oracle/warp_field_oracle.cpp -> oracle/libwarp_oracle.so, built by oracle/Makefile on first use or by oracle.build())
and the serial ICP loop of CombinedMetricDenseWarpFieldICP on the oracle's brute-force 1-NN.

    from oracle import warp_field
    warp_field.icp(dst, dst_n, src, nbhd, max_iter=5, w_pt=0.1, stiffness=200.0)

Transforms are (n, 3, 4) float32 arrays, one [R | t] per source point. nbhd = (offsets, index, value), the CSR of
cb_warp_icp_create.
"""
import ctypes as C

import numpy as np

import oracle
from oracle import FLT_MAX, _p, _rows, rbf_coeff
from oracle import build  # noqa: F401 (oracle.build: every library, also callable as <submodule>.build)


def lib():
    return oracle.load("libwarp_oracle.so",
                       {"orc_warp_solve": C.c_int, "orc_warp_system": C.c_size_t, "orc_warp_huber": C.c_float,
                        "orc_warp_compose": C.c_float},
                       {"orc_warp_huber": [C.c_float, C.c_float, C.c_int],
                        "orc_warp_rotation_terms": [C.c_double, C.c_double, C.c_double, C.c_void_p]})


def _nbhd(nbhd):
    off, idx, val = nbhd
    return (np.ascontiguousarray(off, np.uint64), np.ascontiguousarray(idx, np.int64),
            np.ascontiguousarray(val, np.float32))


def huber(x, delta, derivative=False):
    return float(lib().orc_warp_huber(float(x), float(delta), int(derivative)))


def rotation_terms(a, b, c):
    """computeRotationTerms in double: (rot_coeffs, d/da, d/db, d/dc), each 3x3 as the reference indexes it."""
    out = np.empty(36, np.float64)
    lib().orc_warp_rotation_terms(float(a), float(b), float(c), _p(out))
    return out.reshape(4, 3, 3)


def apply(T, pts):
    """T_i p_i for every point, in the device's float order: (R_r0 x + (R_r1 y + R_r2 z)) + t_r."""
    T = np.asarray(T, np.float32).reshape(-1, 3, 4)
    p = _rows(pts)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    return np.stack([(T[:, r, 0] * x + (T[:, r, 1] * y + T[:, r, 2] * z)) + T[:, r, 3] for r in range(3)], 1)


def system(dst, dst_n, src, first, second, nbhd, x, w_pt=0.0, w_pl=1.0, stiffness=1.0, huber_delta=1e-4,
           reg_sigma=1.0):
    """The normal equations in double at the unknowns x (n, 6): dict(B (n, 21), g (n, 6), diag (n, 6), arc_c, lo, hi)."""
    dst, src = _rows(dst), _rows(src)
    dn = None if dst_n is None else _rows(dst_n)
    n = src.shape[0]
    off, idx, val = _nbhd(nbhd)
    f = np.ascontiguousarray(first, np.uint64)
    s = np.ascontiguousarray(second, np.uint64)
    x = np.ascontiguousarray(x, np.float64).reshape(n, 6)
    args = [_p(dst), _p(dn), C.c_size_t(n), _p(src), C.c_size_t(f.shape[0]), _p(f), _p(s), _p(off), _p(idx), _p(val),
            C.c_size_t(max(off.shape[0] - 1, 0)), C.c_float(w_pt), C.c_float(w_pl), C.c_float(stiffness),
            C.c_float(huber_delta), C.c_float(rbf_coeff(reg_sigma)), _p(x)]
    m = lib().orc_warp_system(*args, None, None, None, None, None, None)
    B = np.empty((n, 21)); g = np.empty((n, 6)); diag = np.empty((n, 6)); c = np.empty((max(m, 1), 6))
    lo = np.empty(max(m, 1), np.uint32); hi = np.empty(max(m, 1), np.uint32)
    lib().orc_warp_system(*args, _p(B), _p(g), _p(diag), _p(c), _p(lo), _p(hi))
    return {"B": B, "g": g, "diag": diag, "arc_c": c[:m], "lo": lo[:m].astype(np.int64), "hi": hi[:m].astype(np.int64)}


def solve(dst, dst_n, src, first, second, nbhd, w_pt=0.0, w_pl=1.0, stiffness=1.0, huber_delta=1e-4, reg_sigma=1.0,
          max_gn_iter=10, gn_tol=1e-5, max_cg_iter=1000, cg_tol=1e-5, double=False):
    """estimateDenseWarpFieldCombinedMetric on src (already transformed). Returns dict(T (n, 3, 4), converged,
    gn_steps, cg_iterations, cg_iterations_last, cg_error, x (n, 6): the unknowns rounded to float)."""
    dst, src = _rows(dst), _rows(src)
    dn = None if dst_n is None else _rows(dst_n)
    n = src.shape[0]
    off, idx, val = _nbhd(nbhd)
    f = np.ascontiguousarray(first, np.uint64)
    s = np.ascontiguousarray(second, np.uint64)
    T = np.empty((max(n, 1), 12), np.float32)
    x = np.empty((max(n, 1), 6), np.float32)
    st = np.zeros(4, np.uint64)
    err = C.c_float()
    lib().orc_warp_solve(C.c_size_t(dst.shape[0]), _p(dst), _p(dn), C.c_size_t(n), _p(src), C.c_size_t(f.shape[0]),
                         _p(f), _p(s), _p(off), _p(idx), _p(val), C.c_size_t(max(off.shape[0] - 1, 0)),
                         C.c_float(w_pt), C.c_float(w_pl), C.c_float(stiffness), C.c_float(huber_delta),
                         C.c_float(rbf_coeff(reg_sigma)), C.c_uint64(int(max_gn_iter)), C.c_float(gn_tol),
                         C.c_uint64(int(max_cg_iter)), C.c_float(cg_tol), C.c_int(int(double)), _p(T), _p(x), _p(st),
                         C.byref(err))
    return {"T": T[:n].reshape(n, 3, 4), "x": x[:n], "converged": bool(st[0]), "gn_steps": int(st[1]),
            "cg_iterations": int(st[2]), "cg_iterations_last": int(st[3]), "cg_error": float(err.value)}


def compose(dT, T):
    """TransformSet::preApply in place on T; returns max_i |dR_i - I|_F^2 + |dt_i|^2."""
    dT = np.ascontiguousarray(dT, np.float32)
    assert T.dtype == np.float32 and T.flags.c_contiguous
    return float(lib().orc_warp_compose(C.c_size_t(dT.shape[0]), _p(dT), _p(T)))


def icp(dst, dst_n, src, nbhd, knn=None, T_init=None, max_iter=15, tol=1e-5, max_d2=1e-4, double=False, **kw):
    """CombinedMetricDenseWarpFieldICP::estimate() (icp_base.hpp:68-87): per iteration the 1-NN of T_i s_i within
    max_d2, the estimator (solve(), kw = its parameters), then T_i <- rotation(dT_i T_i). Returns dict(T, iterations,
    converged, last_delta, num_corr, gn_steps, cg_iterations, first, second)."""
    dst, src = _rows(dst), _rows(src)
    knn = knn or oracle.BruteKnn(dst)
    n = src.shape[0]
    T = np.tile(np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32), (n, 1, 1)) if T_init is None else \
        np.array(T_init, np.float32).reshape(n, 3, 4)
    T = np.ascontiguousarray(T)
    it, last, steps, cgi = 0, float("inf"), 0, 0
    first = second = np.zeros(0, np.int64)
    while it < max_iter:
        q = apply(T, src)
        idx, _ = knn.query(q, max_d2) if dst.shape[0] else (np.full(n, -1), None)
        second = np.nonzero(idx >= 0)[0]
        first = idx[second]
        r = solve(dst, dst_n, q, first, second, nbhd, double=double, **kw)
        steps += r["gn_steps"]
        cgi += r["cg_iterations"]
        last = float(np.sqrt(np.float32(compose(r["T"].reshape(n, 12), T.reshape(n, 12)))))
        it += 1
        if last < tol:
            break
    return {"T": T, "iterations": it, "converged": it > 0 and last < tol, "last_delta": last,
            "num_corr": int(second.shape[0]), "gn_steps": steps, "cg_iterations": cgi, "first": first,
            "second": second}


def residuals(dst, dst_n, src, T, w_pt=0.0, w_pl=1.0):
    """computeResiduals (:216-236) in the device's float order: unbounded 1-NN of T_i s_i,
    w_pt |e|^2 + (w_pl pd) pd with e = d - p, |e|^2 = e0^2 + (e1^2 + e2^2), pd = n0 e0 + (n1 e1 + n2 e2)."""
    dst = _rows(dst)
    q = apply(T, src)
    if dst.shape[0] == 0:
        return np.full(q.shape[0], np.nan, np.float32)
    idx, _ = oracle.BruteKnn(dst).query(q, FLT_MAX)
    e = np.where((idx >= 0)[:, None], dst[np.maximum(idx, 0)], np.float32(np.nan)) - q
    sq = e[:, 0] * e[:, 0] + (e[:, 1] * e[:, 1] + e[:, 2] * e[:, 2])
    if dst_n is None:
        return np.float32(w_pt) * sq
    nn = _rows(dst_n)[np.maximum(idx, 0)]
    pd = nn[:, 0] * e[:, 0] + (nn[:, 1] * e[:, 1] + nn[:, 2] * e[:, 2])
    return np.float32(w_pt) * sq + (np.float32(w_pl) * pd) * pd
