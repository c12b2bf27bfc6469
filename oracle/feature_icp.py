"""ORACLE — test infrastructure, NOT product code: the feature-space rigid ICP restated on the CPU
(oracle/feature_icp_oracle.cpp -> oracle/libfeature_icp_oracle.so) and, where the reference exists, its own nanoflann
on D = 3 / 6 / 9 feature vectors (oracle/nanoflann_feature_ref.cpp -> oracle/_ref/libcilantro_ref_feature_knn.so).
Both are built by oracle/Makefile (oracle.build()).

    from oracle import feature_icp
    dt = feature_icp.tails("point_color", None, dst_colors, 1.0, 5.0)
    st = feature_icp.tails("point_color", None, src_colors, 1.0, 5.0)
    out = feature_icp.icp("point_color", dst, dt, src, st, metric="p2p", max_d2=1e-3)

Tails are the weighted feature parts after xyz, (n, 3 * tails) float32: w_n n and / or w_c c.
"""
import ctypes as C

import numpy as np

import oracle
from oracle import _p, _rows
from oracle import build  # noqa: F401 (oracle.build: every library, also callable as <submodule>.build)

KINDS = {"point": 0, "point_normal": 1, "point_color": 2, "point_normal_color": 3}


def lib():
    return oracle.load("libfeature_icp_oracle.so", {"orc_feature_engine_correspondences": C.c_size_t})


def ref():
    """The reference's own nanoflann over feature vectors (None without oracle/_ref)."""
    return oracle.load("_ref/libcilantro_ref_feature_knn.so")


def have_ref():
    return ref() is not None


def ntails(kind):
    return {0: 0, 1: 1, 2: 1, 3: 2}[KINDS[kind]]


def tails(kind, normals, colors, w_n=1.0, w_c=1.0):
    """The feature parts after xyz: (n, 3 * tails), w_n n then w_c c."""
    src = normals if normals is not None else colors
    n = np.asarray(src).reshape(-1, 3).shape[0]
    nrm = _rows(normals, 3) if normals is not None else None
    col = _rows(colors, 3) if colors is not None else None
    out = np.empty((n, 3 * ntails(kind)), np.float32)
    lib().orc_feature_tails(C.c_int(KINDS[kind]), _p(nrm), _p(col), C.c_size_t(n), C.c_float(w_n), C.c_float(w_c),
                            _p(out))
    return out


def features(kind, T, xyz, tl):
    """transformFeatures(T): packed (n, D) features."""
    xyz = _rows(xyz, 3)
    nt = ntails(kind)
    tl = _rows(tl, 3 * nt) if nt else np.zeros((xyz.shape[0], 0), np.float32)
    out = np.empty((xyz.shape[0], 3 + 3 * nt), np.float32)
    lib().orc_transform_features(C.c_int(KINDS[kind]), _p(oracle._T(T)), _p(xyz), _p(tl), C.c_size_t(xyz.shape[0]),
                                 _p(out))
    return out


def knn1(ref_feats, qry_feats, max_d2):
    """Brute-force radius-bounded 1-NN of packed features (lowest index on exact ties): idx (-1 = none), d2."""
    D = ref_feats.shape[1]
    r, q = _rows(ref_feats, D), _rows(qry_feats, D)
    idx = np.empty(q.shape[0], np.int64)
    d2 = np.empty(q.shape[0], np.float32)
    lib().orc_feature_knn1(_p(r), C.c_size_t(r.shape[0]), _p(q), C.c_size_t(q.shape[0]), C.c_size_t(D),
                           C.c_float(max_d2), _p(idx), _p(d2))
    return idx, d2


def ref_knn1(ref_feats, qry_feats, max_d2):
    """The same search through the reference's nanoflann kd-tree (ties: traversal order)."""
    D = ref_feats.shape[1]
    r, q = _rows(ref_feats, D), _rows(qry_feats, D)
    idx = np.empty(q.shape[0], np.int64)
    d2 = np.empty(q.shape[0], np.float32)
    assert ref().ref_feature_knn1(C.c_size_t(D), _p(r), C.c_size_t(r.shape[0]), _p(q), C.c_size_t(q.shape[0]),
                                  C.c_float(max_d2), _p(idx), _p(d2)) == 0
    return idx, d2


def ref_l2_eval(a, b):
    """nanoflann's L2_Adaptor::evalMetric on row pairs of packed (n, D) vectors."""
    D = a.shape[1]
    a, b = _rows(a, D), _rows(b, D)
    out = np.empty(a.shape[0], np.float32)
    assert ref().ref_l2_eval(C.c_size_t(D), _p(a), _p(b), C.c_size_t(a.shape[0]), _p(out)) == 0
    return out


def _tl(kind, tl, n):
    nt = ntails(kind)
    return _rows(tl, 3 * nt) if nt else np.zeros((n, 0), np.float32)


def engine_correspondences(kind, dst, dst_tails, src, src_tails, T, max_d2, search_dir="second_to_first",
                           inlier_fraction=1.0, require_reciprocal=False, one_to_one=False):
    """findCorrespondences(T).getCorrespondences() of the feature engine: (first, second, value)."""
    dst, src = _rows(dst, 3), _rows(src, 3)
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
    dst, src = _rows(dst, 3), _rows(src, 3)
    dt, st = _tl(kind, dst_tails, dst.shape[0]), _tl(kind, src_tails, src.shape[0])
    dn = _rows(dst_n, 3) if dst_n is not None else None
    sn = _rows(src_n, 3) if src_n is not None else None
    prm = oracle._icp_params(metric, max_iter, tol, max_d2, w_pt, w_pl, max_opt_iter, opt_tol, T_init, pt_rbf_sigma,
                             pl_rbf_sigma, search_dir=search_dir, inlier_fraction=inlier_fraction,
                             require_reciprocal=require_reciprocal, one_to_one=one_to_one)
    if prm.metric == 1:
        assert dn is not None
    res = oracle.IcpResult()
    lib().orc_feature_icp(C.c_int(KINDS[kind]), _p(dst), _p(dn), _p(dt), C.c_size_t(dst.shape[0]), _p(src), _p(sn),
                          _p(st), C.c_size_t(src.shape[0]), C.byref(prm), C.byref(res), None)
    return {"T": np.array(list(res.T), np.float32).reshape(3, 4), "iterations": int(res.iterations),
            "num_corr": int(res.last_num_corr), "last_delta": float(res.last_delta), "converged": bool(res.converged)}
