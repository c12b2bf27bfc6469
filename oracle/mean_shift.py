"""ORACLE — test infrastructure, NOT product code: ctypes binding of the mean-shift restatement
(oracle/mean_shift_oracle.cpp -> oracle/libms_oracle.so, built by oracle/Makefile on first use or by oracle.build()).

    from oracle import mean_shift
    mean_shift.mean_shift(pts, kernel_radius=2.0, max_iter=100, cluster_tol=0.2)

The result dict has the layout of capi.Cloud.mean_shift.
"""
import ctypes as C

import numpy as np

import oracle
from oracle import _p, _rows, rbf_coeff
from oracle import build  # noqa: F401 (oracle.build: every library, also callable as <submodule>.build)

FLT_EPSILON = float(np.finfo(np.float32).eps)


def lib():
    return oracle.load("libms_oracle.so", {"orc_mean_shift": C.c_uint64})


def mean_shift(pts, kernel_radius, max_iter, cluster_tol, convergence_tol=FLT_EPSILON, seeds=None, weight="unity"):
    """MeanShift3f::cluster restated serially per seed. seeds None = the points themselves; weight "unity" or
    ("rbf", sigma). Returns dict(offsets, points, point_to_cluster, num_clusters, shifted_seeds, modes, iterations)."""
    pts = _rows(pts)
    sd = pts if seeds is None else _rows(seeds)
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
