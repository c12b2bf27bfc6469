"""ORACLE — test infrastructure, NOT product code: ctypes binding of the mean-shift restatement
(oracle/mean_shift_oracle.cpp -> oracle/libms_oracle.so, built on first use or by build()).

    from oracle import mean_shift
    mean_shift.mean_shift(pts, kernel_radius=2.0, max_iter=100, cluster_tol=0.2)

The result dict has the layout of capi.Cloud.mean_shift.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "mean_shift_oracle.cpp")
_LIB_PATH = os.path.join(_HERE, "libms_oracle.so")
_lib = None

FLT_EPSILON = float(np.finfo(np.float32).eps)


def build(force=False):
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(_SRC):
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
        _lib.orc_mean_shift.restype = C.c_uint64
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def rbf_coeff(sigma):
    """RBFKernelWeightEvaluator's coefficient in float: -(0.5f) / (sigma * sigma)."""
    sg = np.float32(sigma)
    return float(np.float32(-0.5) / (sg * sg))


def mean_shift(pts, kernel_radius, max_iter, cluster_tol, convergence_tol=FLT_EPSILON, seeds=None, weight="unity"):
    """MeanShift3f::cluster restated serially per seed. seeds None = the points themselves; weight "unity" or
    ("rbf", sigma). Returns dict(offsets, points, point_to_cluster, num_clusters, shifted_seeds, modes, iterations)."""
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    sd = pts if seeds is None else np.ascontiguousarray(seeds, np.float32).reshape(-1, 3)
    ns = sd.shape[0]
    rbf, coeff = (0, 0.0) if weight == "unity" else (1, rbf_coeff(weight[1]))
    shifted = np.empty((max(ns, 1), 3), np.float32)
    modes = np.empty((max(ns, 1), 3), np.float32)
    p2c = np.empty(max(ns, 1), np.uint64)
    off = np.empty(ns + 1, np.uint64)
    mem = np.empty(max(ns, 1), np.uint64)
    m = C.c_size_t()
    it = lib().orc_mean_shift(C.c_size_t(pts.shape[0]), _p(pts), C.c_size_t(ns), _p(sd if ns else shifted),
                              C.c_float(kernel_radius), C.c_uint64(int(max_iter)), C.c_float(cluster_tol),
                              C.c_float(convergence_tol), C.c_int(rbf), C.c_float(coeff), _p(shifted), _p(p2c), _p(off),
                              _p(mem), _p(modes), C.byref(m))
    m = m.value
    off = off[:m + 1].astype(np.int64)
    return {"offsets": off, "points": mem[:off[-1]].astype(np.int64), "point_to_cluster": p2c[:ns].astype(np.int64),
            "num_clusters": m, "shifted_seeds": shifted[:ns].copy(), "modes": modes[:m].copy(), "iterations": int(it)}
