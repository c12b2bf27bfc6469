"""ORACLE — test infrastructure, NOT product code: ctypes binding of the plane-RANSAC restatement
(oracle/plane_ransac_oracle.cpp -> oracle/libplane_oracle.so, built by oracle/Makefile on first use or by
oracle.build()).

    from oracle import ransac_plane
    ransac_plane.ransac_plane(pts, seed=3, max_iter=250, thresh=0.01, inlier_count_thresh=1500)

Planes are float32 (n0, n1, n2, d). The result dict of ransac_plane() has the keys of capi.ransac_plane's.
"""
import ctypes as C

import numpy as np

import oracle
from oracle import _p, _rows
from oracle import build  # noqa: F401 (oracle.build: every library, also callable as <submodule>.build)


class PlaneResult(C.Structure):
    _fields_ = [
        ("plane", C.c_float * 4),
        ("hyp_plane", C.c_float * 4),
        ("iterations", C.c_uint64),
        ("best_iteration", C.c_uint64),
        ("num_inliers", C.c_uint64),
    ]


def lib():
    return oracle.load("libplane_oracle.so", {"orc_plane_residuals": C.c_size_t})


def fit(sample_points):
    """The hypothesis plane of a sample of 0..3 points (DESIGN §4.12)."""
    p = np.zeros(9, np.float32)
    s = np.asarray(sample_points, np.float32).reshape(-1)
    p[:s.size] = s
    out = np.empty(4, np.float32)
    lib().orc_plane_fit(_p(p), C.c_int(s.size // 3), _p(out))
    return out


def residuals(pts, plane, thresh):
    """(residuals[n], ascending inlier indices) of one plane."""
    pts = _rows(pts)
    pl = np.ascontiguousarray(plane, np.float32).reshape(4)
    n = pts.shape[0]
    res = np.empty(max(n, 1), np.float32)
    inl = np.empty(max(n, 1), np.uint64)
    k = lib().orc_plane_residuals(_p(pts), C.c_size_t(n), _p(pl), C.c_float(thresh), _p(res), _p(inl))
    return res[:n].copy(), inl[:k].astype(np.int64)


def score(pts, planes, thresh):
    pts = _rows(pts)
    planes = np.ascontiguousarray(planes, np.float32).reshape(-1, 4)
    counts = np.empty(planes.shape[0], np.uint32)
    lib().orc_plane_score(_p(pts), C.c_size_t(pts.shape[0]), _p(planes), C.c_size_t(planes.shape[0]), C.c_float(thresh),
                          _p(counts))
    return counts


def hypotheses(pts, seed, iters):
    """The loop's first `iters` samples (iters x min(3, n) indices) and their planes (iters x 4)."""
    pts = _rows(pts)
    n = pts.shape[0]
    samples = np.zeros((iters, 3), np.uint64)
    planes = np.empty((max(iters, 1), 4), np.float32)
    lib().orc_plane_hypotheses(_p(pts), C.c_size_t(n), C.c_uint32(seed), C.c_size_t(iters), _p(samples), _p(planes))
    return samples[:, :min(n, 3)].astype(np.int64), planes[:iters].copy()


def pca_plane(pts, idx, accum_double=False):
    """estimateModel(sample_ind): the PCA plane of the listed points."""
    pts = _rows(pts)
    idx = np.ascontiguousarray(idx, np.uint64)
    out = np.empty(4, np.float32)
    lib().orc_plane_pca(_p(pts), _p(idx), C.c_size_t(idx.size), C.c_int(int(accum_double)), _p(out))
    return out


def ransac_plane(pts, seed, max_iter=100, thresh=0.1, inlier_count_thresh=None, re_estimate=True, accum_double=False):
    """PlaneRANSACEstimator3f::estimate restated serially, the seed injected in place of std::random_device."""
    pts = _rows(pts)
    n = pts.shape[0]
    if inlier_count_thresh is None:
        inlier_count_thresh = n // 2 + n % 2  # ransac_hyperplane_estimator.hpp:18
    res = PlaneResult()
    inl = np.empty(max(n, 1), np.uint64)
    resid = np.empty(max(n, 1), np.float32)
    lib().orc_ransac_plane(_p(pts), C.c_size_t(n), C.c_uint32(seed), C.c_size_t(inlier_count_thresh),
                           C.c_size_t(max_iter), C.c_float(thresh), C.c_int(int(re_estimate)), C.c_int(int(accum_double)),
                           C.byref(res), _p(inl), _p(resid))
    return {"plane": np.array(list(res.plane), np.float32), "hyp_plane": np.array(list(res.hyp_plane), np.float32),
            "iterations": int(res.iterations), "best_iteration": int(res.best_iteration),
            "num_inliers": int(res.num_inliers), "inliers": inl[:res.num_inliers].astype(np.int64),
            "residuals": resid[:n].copy()}
