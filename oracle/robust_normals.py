"""ORACLE — test infrastructure, NOT product code: ctypes binding of the robust-normal restatement
(oracle/robust_normals_oracle.cpp -> oracle/librobust_normals_oracle.so, built on first use or by build()).

    from oracle import robust_normals
    out = robust_normals.estimate_normals_mcd(pts, k=12, chi_square_threshold=6.25, num_trials=2, num_refinements=1)

Neighbourhoods come from the brute-force search of the main oracle (ascending (d2, index)). The result dict has the keys
of capi.Cloud.estimate_normals_mcd's, plus "kept" (the winning trial's kept neighbour indices, -1 padded), "h" and
"nbr" / "cnt" (the neighbourhoods).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "robust_normals_oracle.cpp")
_DEPS = (_SRC, os.path.join(_HERE, "small_linalg.hpp"))
_LIB_PATH = os.path.join(_HERE, "librobust_normals_oracle.so")
_lib = None


def build(force=False):
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < max(os.path.getmtime(d) for d in _DEPS):
        env = dict(os.environ)
        env.pop("CXX", None)
        tmp = _LIB_PATH + f".{os.getpid()}.tmp"
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fopenmp", "-fPIC",
                               "-shared", "-fvisibility=hidden", "-Wall", "-o", tmp, _SRC], env=env)
        os.replace(tmp, _LIB_PATH)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        _lib = C.CDLL(_LIB_PATH)
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def estimate_normals_mcd(pts, k, radius2=0.0, view_point=None, ref_normals=None, num_trials=6, num_refinements=3,
                         inlier_ratio=0.75, chi_square_threshold=-1.0, min_sample_size=3, seed=0, neighbors=None):
    """NormalEstimation<float, 3, MinimumCovarianceDeterminant<float, 3>>::estimateNormalsAndCurvature{KNN,KNNInRadius}
    restated serially, the draws seeded per point as in DESIGN §4.15. neighbors = (idx, cnt) skips the search."""
    import oracle

    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    n = pts.shape[0]
    if neighbors is None:
        max_d2 = float(radius2) if radius2 > 0 else 3.402823466e38
        idx, _, cnt = oracle.BruteKnn(pts).neighborhoods(pts, k, max_d2, stride=k)
    else:
        idx, cnt = neighbors
    idx = np.ascontiguousarray(idx, np.int64).reshape(n, -1)
    cnt = np.ascontiguousarray(cnt, np.uint32)
    stride = idx.shape[1]
    vp = None if view_point is None else np.ascontiguousarray(view_point, np.float32).reshape(3)
    rn = None if ref_normals is None else np.ascontiguousarray(ref_normals, np.float32).reshape(-1, 3)
    normals = np.empty((n, 3), np.float32)
    curv = np.empty(n, np.float32)
    cov6 = np.empty((n, 6), np.float32)
    status = np.empty(n, np.uint8)
    kept = np.empty((n, stride), np.int32)
    h = np.empty(n, np.uint32)
    lib().orc_mcd_normals(_p(pts), C.c_size_t(n), _p(idx), C.c_size_t(stride), _p(cnt), C.c_int(num_trials),
                          C.c_int(num_refinements), C.c_float(inlier_ratio), C.c_float(chi_square_threshold),
                          C.c_int(min_sample_size), C.c_uint32(int(seed) & 0xFFFFFFFF), _p(vp), _p(rn), _p(normals),
                          _p(curv), _p(cov6), _p(status), _p(kept), _p(h))
    return {"normals": normals, "curvature": curv, "cov6": cov6, "status": status, "kept": kept, "h": h, "nbr": idx,
            "cnt": cnt}
