"""ORACLE — test infrastructure, NOT product code: the feature-space rigid ICP restated on the CPU
(oracle/feature_icp_oracle.cpp -> oracle/libfeature_icp_oracle.so) and, where the reference exists, its own nanoflann
on D = 3 / 6 / 9 feature vectors (oracle/nanoflann_feature_ref.cpp -> oracle/_ref/libcilantro_ref_feature_knn.so).
Both are built by build() (called from __graft_entry__.build()).

    from oracle import feature_icp
    dt = feature_icp.tails("point_color", None, dst_colors, 1.0, 5.0)
    st = feature_icp.tails("point_color", None, src_colors, 1.0, 5.0)
    out = feature_icp.icp("point_color", dst, dt, src, st, metric="p2p", max_d2=1e-3)

Tails are the weighted feature parts after xyz, (n, 3 * tails) float32: w_n n and / or w_c c.
"""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "feature_icp_oracle.cpp")
_DEPS = (_SRC, os.path.join(_HERE, "cilantro_oracle.cpp"), os.path.join(_HERE, "small_linalg.hpp"))
_LIB_PATH = os.path.join(_HERE, "libfeature_icp_oracle.so")
_REF_SRC = os.path.join(_HERE, "nanoflann_feature_ref.cpp")
_REF_DEPS = (_REF_SRC, os.path.join(_HERE, "nanoflann_ref.cpp"))
_REF_PATH = os.path.join(_HERE, "_ref", "libcilantro_ref_feature_knn.so")
_NANOFLANN = "/root/reference/include/cilantro/3rd_party/nanoflann"
_FLAGS = ["-std=c++17", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared",
          "-fvisibility=hidden", "-Wall"]

KINDS = {"point": 0, "point_normal": 1, "point_color": 2, "point_normal_color": 3}
_lib = None
_ref = None


def _stale(target, deps):
    return not os.path.exists(target) or os.path.getmtime(target) < max(os.path.getmtime(d) for d in deps)


def _compile(target, src, extra=()):
    env = dict(os.environ)
    env.pop("CXX", None)
    os.makedirs(os.path.dirname(target), exist_ok=True)
    tmp = target + f".{os.getpid()}.tmp"
    subprocess.check_call(["g++"] + _FLAGS + list(extra) + ["-o", tmp, src], env=env)
    os.replace(tmp, target)


def build(force=False):
    if force or _stale(_LIB_PATH, _DEPS):
        _compile(_LIB_PATH, _SRC)
    if os.path.exists(os.path.join(_NANOFLANN, "nanoflann.hpp")) and (force or _stale(_REF_PATH, _REF_DEPS)):
        _compile(_REF_PATH, _REF_SRC, ["-I", _NANOFLANN])


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_feature_engine_correspondences.restype = C.c_size_t
    return _lib


def have_ref():
    return os.path.exists(_REF_PATH)


def ref():
    """The reference's own nanoflann over feature vectors (None if oracle/_ref was never built)."""
    global _ref
    if _ref is None and have_ref():
        _ref = C.CDLL(_REF_PATH)
    return _ref


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _f32(a, cols):
    a = np.ascontiguousarray(a, np.float32)
    return a.reshape(-1, cols)


def ntails(kind):
    return {0: 0, 1: 1, 2: 1, 3: 2}[KINDS[kind]]


def tails(kind, normals, colors, w_n=1.0, w_c=1.0):
    """The feature parts after xyz: (n, 3 * tails), w_n n then w_c c."""
    src = normals if normals is not None else colors
    n = np.asarray(src).reshape(-1, 3).shape[0]
    nrm = _f32(normals, 3) if normals is not None else None
    col = _f32(colors, 3) if colors is not None else None
    out = np.empty((n, 3 * ntails(kind)), np.float32)
    lib().orc_feature_tails(C.c_int(KINDS[kind]), _p(nrm), _p(col), C.c_size_t(n), C.c_float(w_n), C.c_float(w_c),
                            _p(out))
    return out


def features(kind, T, xyz, tl):
    """transformFeatures(T): packed (n, D) features."""
    xyz = _f32(xyz, 3)
    nt = ntails(kind)
    tl = _f32(tl, 3 * nt) if nt else np.zeros((xyz.shape[0], 0), np.float32)
    out = np.empty((xyz.shape[0], 3 + 3 * nt), np.float32)
    lib().orc_transform_features(C.c_int(KINDS[kind]), _p(oracle._T(T)), _p(xyz), _p(tl), C.c_size_t(xyz.shape[0]),
                                 _p(out))
    return out


def knn1(ref_feats, qry_feats, max_d2):
    """Brute-force radius-bounded 1-NN of packed features (lowest index on exact ties): idx (-1 = none), d2."""
    D = ref_feats.shape[1]
    r, q = _f32(ref_feats, D), _f32(qry_feats, D)
    idx = np.empty(q.shape[0], np.int64)
    d2 = np.empty(q.shape[0], np.float32)
    lib().orc_feature_knn1(_p(r), C.c_size_t(r.shape[0]), _p(q), C.c_size_t(q.shape[0]), C.c_size_t(D),
                           C.c_float(max_d2), _p(idx), _p(d2))
    return idx, d2


def ref_knn1(ref_feats, qry_feats, max_d2):
    """The same search through the reference's nanoflann kd-tree (ties: traversal order)."""
    D = ref_feats.shape[1]
    r, q = _f32(ref_feats, D), _f32(qry_feats, D)
    idx = np.empty(q.shape[0], np.int64)
    d2 = np.empty(q.shape[0], np.float32)
    assert ref().ref_feature_knn1(C.c_size_t(D), _p(r), C.c_size_t(r.shape[0]), _p(q), C.c_size_t(q.shape[0]),
                                  C.c_float(max_d2), _p(idx), _p(d2)) == 0
    return idx, d2


def ref_l2_eval(a, b):
    """nanoflann's L2_Adaptor::evalMetric on row pairs of packed (n, D) vectors."""
    D = a.shape[1]
    a, b = _f32(a, D), _f32(b, D)
    out = np.empty(a.shape[0], np.float32)
    assert ref().ref_l2_eval(C.c_size_t(D), _p(a), _p(b), C.c_size_t(a.shape[0]), _p(out)) == 0
    return out


def _tl(kind, tl, n):
    nt = ntails(kind)
    return _f32(tl, 3 * nt) if nt else np.zeros((n, 0), np.float32)


def engine_correspondences(kind, dst, dst_tails, src, src_tails, T, max_d2, search_dir="second_to_first",
                           inlier_fraction=1.0, require_reciprocal=False, one_to_one=False):
    """findCorrespondences(T).getCorrespondences() of the feature engine: (first, second, value)."""
    dst, src = _f32(dst, 3), _f32(src, 3)
    dt, st = _tl(kind, dst_tails, dst.shape[0]), _tl(kind, src_tails, src.shape[0])
    prm = oracle.IcpParams()
    prm.max_d2 = max_d2
    oracle._engine_fields(prm, search_dir, inlier_fraction, require_reciprocal, one_to_one)
    cap = dst.shape[0] + src.shape[0]
    i1 = np.empty(cap, np.uint64)
    i2 = np.empty(cap, np.uint64)
    v = np.empty(cap, np.float32)
    m = lib().orc_feature_engine_correspondences(C.c_int(KINDS[kind]), _p(dst), _p(dt), C.c_size_t(dst.shape[0]),
                                                 _p(src), _p(st), C.c_size_t(src.shape[0]), _p(oracle._T(T)),
                                                 C.byref(prm), _p(i1), _p(i2), _p(v))
    return i1[:m].astype(np.int64), i2[:m].astype(np.int64), v[:m].copy()


def icp(kind, dst, dst_tails, src, src_tails, metric="p2p", dst_n=None, src_n=None, max_iter=15, tol=1e-5,
        max_d2=1e-4, w_pt=0.0, w_pl=1.0, max_opt_iter=1, opt_tol=1e-5, T_init=None, search_dir="second_to_first",
        inlier_fraction=1.0, require_reciprocal=False, one_to_one=False, pt_rbf_sigma=None, pl_rbf_sigma=None):
    """oracle.icp with the feature search (every configuration on the list path). Returns a dict."""
    dst, src = _f32(dst, 3), _f32(src, 3)
    dt, st = _tl(kind, dst_tails, dst.shape[0]), _tl(kind, src_tails, src.shape[0])
    dn = _f32(dst_n, 3) if dst_n is not None else None
    sn = _f32(src_n, 3) if src_n is not None else None
    prm = oracle.IcpParams()
    oracle._engine_fields(prm, search_dir, inlier_fraction, require_reciprocal, one_to_one)
    prm.metric = 0 if metric == "p2p" else 1
    prm.max_iter, prm.tol, prm.max_d2 = int(max_iter), tol, max_d2
    prm.w_pt, prm.w_pl = w_pt, w_pl
    prm.max_opt_iter, prm.opt_tol = int(max_opt_iter), opt_tol
    for k, c, sigma in (("pt_weight_kind", "pt_weight_coeff", pt_rbf_sigma),
                        ("pl_weight_kind", "pl_weight_coeff", pl_rbf_sigma)):
        if sigma is not None:
            sg = np.float32(sigma)
            setattr(prm, k, 1)
            setattr(prm, c, float(np.float32(-0.5) / (sg * sg)))
    Ti = oracle.identity() if T_init is None else oracle._T(T_init)
    for i, v in enumerate(Ti.reshape(-1)):
        prm.T_init[i] = float(v)
    if prm.metric == 1:
        assert dn is not None
    res = oracle.IcpResult()
    lib().orc_feature_icp(C.c_int(KINDS[kind]), _p(dst), _p(dn), _p(dt), C.c_size_t(dst.shape[0]), _p(src), _p(sn),
                          _p(st), C.c_size_t(src.shape[0]), C.byref(prm), C.byref(res), None)
    return {"T": np.array(list(res.T), np.float32).reshape(3, 4), "iterations": int(res.iterations),
            "num_corr": int(res.last_num_corr), "last_delta": float(res.last_delta), "converged": bool(res.converged)}
