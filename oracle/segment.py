"""ORACLE — test infrastructure, NOT product code: ctypes binding of the connected-component restatement
(oracle/cce_oracle.cpp -> oracle/libcce_oracle.so, built by oracle/Makefile on first use or by oracle.build()).

    from oracle import segment
    segment.connected_components(pts, k=0, radius2=r2, terms=2, max_angle=a, normals=nrm)

Neighbourhoods: BruteKnn (oracle/cilantro_oracle.cpp, ascending (d2, index)) by default, or any object with the
same neighborhoods(qry, k, r2, stride) method whose rows are re-sorted on (d2, index) here (e.g. RefKnn).
"""
import ctypes as C

import numpy as np

import oracle
from oracle import FLT_MAX, _p
from oracle import build  # noqa: F401 (oracle.build: every library, also callable as <submodule>.build)


def lib():
    return oracle.load("libcce_oracle.so", {"orc_connected_components": C.c_size_t})


def neighborhoods(pts, k=0, radius2=0.0, knn=None):
    """N(p) of every point over the cloud itself, ascending (d2, index): (idx [n, stride], d2, cnt).
    Encoding of cb_cloud_estimate_normals: k > 0, radius2 <= 0: kNN; k > 0, radius2 > 0: kNN in radius; k == 0: radius."""
    pts = np.ascontiguousarray(pts, np.float32)
    knn = knn if knn is not None else oracle.BruteKnn(pts)
    r2 = float(radius2) if radius2 > 0 else FLT_MAX
    n = pts.shape[0]
    if n == 0:
        return np.zeros((0, 1), np.int64), np.zeros((0, 1), np.float32), np.zeros(0, np.uint32)
    if k > 0:
        idx, d2, cnt = knn.neighborhoods(pts, k, r2)
    else:
        _, _, cnt = knn.neighborhoods(pts, 0, r2, stride=1)
        idx, d2, cnt = knn.neighborhoods(pts, 0, r2, stride=max(1, int(cnt.max())))
    if knn.kind != "port":
        idx, d2 = sort_rows(idx, d2, cnt)
    return idx, d2, cnt


def sort_rows(idx, d2, cnt):
    """Re-sorts every row's valid entries on (d2, index), the pinned order of equal distances (the reference's kd-tree
    returns equal distances in traversal order); padding moves to the end of each row."""
    n, s = idx.shape
    valid = np.arange(s)[None, :] < cnt[:, None].astype(np.int64)
    ki = np.where(valid, idx, np.iinfo(np.int64).max).ravel()
    kd = np.where(valid, d2, np.float32(np.inf)).ravel()
    o = np.lexsort((ki, kd, np.repeat(np.arange(n), s)))
    return ki[o].reshape(n, s), kd[o].reshape(n, s)


def connected_components(pts, k=0, radius2=0.0, terms=0, max_distance=0.0, max_angle=0.0, color_thresh=0.0,
                         angle_strict=False, normals=None, colors=None, seeds=None, min_size=1, max_size=2**64 - 1,
                         knn=None, nbhd=None):
    """extractConnectedComponents (one thread, stable size sort). Returns dict(offsets, points, point_to_cluster,
    num_clusters) in the layout of capi.Cloud.segment. nbhd = precomputed (idx, d2, cnt) rows."""
    pts = np.ascontiguousarray(pts, np.float32)
    n = pts.shape[0]
    idx, d2, cnt = nbhd if nbhd is not None else neighborhoods(pts, k, radius2, knn)
    idx = np.ascontiguousarray(idx, np.int64)
    d2 = np.ascontiguousarray(d2, np.float32)
    cnt = np.ascontiguousarray(cnt, np.uint32)
    nrm = np.ascontiguousarray(normals, np.float32) if normals is not None else None
    col = np.ascontiguousarray(colors, np.float32) if colors is not None else None
    sd = np.ascontiguousarray(seeds, np.uint64) if seeds is not None else None
    if sd is not None and sd.size == 0:
        sd = np.zeros(1, np.uint64)
        n_seeds = 0
    else:
        n_seeds = 0 if sd is None else sd.size
    p2c = np.empty(max(n, 1), np.uint64)
    off = np.empty(n + 1, np.uint64)
    out = np.empty(max(n, 1), np.uint64)
    m = lib().orc_connected_components(
        C.c_size_t(n), _p(idx), _p(d2), C.c_size_t(idx.shape[1] if idx.ndim == 2 else 1), _p(cnt), _p(sd),
        C.c_size_t(n_seeds), C.c_int(int(terms)), C.c_int(int(bool(angle_strict))), C.c_float(max_distance),
        C.c_float(max_angle), C.c_float(color_thresh), _p(nrm), _p(col), C.c_uint64(int(min_size)),
        C.c_uint64(int(max_size)), _p(p2c), _p(off), _p(out))
    off = off[:m + 1].astype(np.int64)
    return {"offsets": off, "points": out[:off[-1]].astype(np.int64), "point_to_cluster": p2c[:n].astype(np.int64),
            "num_clusters": int(m)}
