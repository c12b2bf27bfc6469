"""ORACLE — test infrastructure, NOT product code.

ctypes bindings for the CPU restatement (oracle/libcilantro_oracle.so, built from
cilantro_oracle.cpp) and, when present, for the reference's own vendored nanoflann compiled in
place (oracle/_ref/libcilantro_ref_knn.so, built from nanoflann_ref.cpp against the
reference checkout). Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs may import this package; cilantro_b200 never does.

oracle/Makefile builds every library of the package (build()); load() opens one for this module
and each submodule. The ctypes helpers they share live here.

All point sets are numpy float32 arrays of shape (n, 3), C-contiguous — byte-identical to the
reference's column-major 3 x n Eigen layout (core/data_containers.hpp:155-156).
Transforms are float32 (3, 4) row-major [R | t].
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))

KNN_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_size_t, C.c_float, C.c_void_p, C.c_void_p)
FLT_MAX = float(np.finfo(np.float32).max)


def build(force=False):
    """Compile every oracle library that is missing or stale (oracle/Makefile: the restatements, and the reference's
    nanoflann into oracle/_ref where a reference checkout exists); force rebuilds them all."""
    global _built
    subprocess.check_call(["make", "-s", "-C", _HERE, f"-j{os.cpu_count() or 1}"] + (["-B"] if force else []))
    _built = True


_built = False
_libs = {}


def load(name, restype=None, argtypes=None):
    """The library oracle/<name>, opened once per process after one build() (a no-op when nothing is stale), with the
    given {function: restype} and {function: argtypes} set. None if the build leaves no such file (oracle/_ref without
    a reference checkout)."""
    if name not in _libs:
        if not _built:
            build()
        path = os.path.join(_HERE, name)
        h = C.CDLL(path) if os.path.exists(path) else None
        if h is not None:
            for fn, t in (restype or {}).items():
                getattr(h, fn).restype = t
            for fn, t in (argtypes or {}).items():
                getattr(h, fn).argtypes = t
        _libs[name] = h
    return _libs[name]


class IcpParams(C.Structure):
    _fields_ = [
        ("metric", C.c_int32),
        ("max_iter", C.c_int32),
        ("tol", C.c_float),
        ("max_d2", C.c_float),
        ("w_pt", C.c_float),
        ("w_pl", C.c_float),
        ("max_opt_iter", C.c_int32),
        ("opt_tol", C.c_float),
        ("accum_double", C.c_int32),
        ("parallel", C.c_int32),
        ("T_init", C.c_float * 12),
        ("search_dir", C.c_int32),
        ("require_reciprocal", C.c_int32),
        ("one_to_one", C.c_int32),
        ("reserved_", C.c_int32),
        ("inlier_fraction", C.c_double),
        ("f2s_fn", C.c_void_p),
        ("pt_weight_kind", C.c_int32),
        ("pl_weight_kind", C.c_int32),
        ("pt_weight_coeff", C.c_float),
        ("pl_weight_coeff", C.c_float),
    ]


SEARCH_DIR = {"second_to_first": 0, "first_to_second": 1, "both": 2}


class IcpResult(C.Structure):
    _fields_ = [
        ("T", C.c_float * 12),
        ("iterations", C.c_int32),
        ("last_delta", C.c_float),
        ("converged", C.c_int32),
        ("last_num_corr", C.c_uint64),
        ("t_knn_s", C.c_double),
        ("t_est_s", C.c_double),
    ]


class RansacResult(C.Structure):
    _fields_ = [
        ("T", C.c_float * 12),
        ("iterations", C.c_uint64),
        ("num_inliers", C.c_uint64),
        ("best_iteration", C.c_uint64),
    ]


class BruteCtx(C.Structure):
    _fields_ = [("ref", C.c_void_p), ("nref", C.c_size_t)]


def lib():
    return load("libcilantro_oracle.so", {"orc_kmeans": C.c_size_t, "orc_find_correspondences": C.c_size_t,
                                          "orc_num_threads": C.c_int, "orc_engine_correspondences": C.c_size_t,
                                          "orc_grid_downsample": C.c_size_t})


def ref():
    """The reference's own nanoflann (None without oracle/_ref)."""
    return load("_ref/libcilantro_ref_knn.so", {"ref_tree_build": C.c_void_p, "ref_knn_in_radius": C.c_size_t,
                                                "ref_nanoflann_version": C.c_uint})


def have_ref():
    return ref() is not None


def _f32(a, shape_last=3):
    """float32, C-contiguous; asserts the shape (n, shape_last) unless shape_last is None."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    if shape_last is not None:
        assert a.ndim == 2 and a.shape[1] == shape_last, a.shape
    return a


def _rows(a, cols=3):
    """float32, C-contiguous, reshaped to (-1, cols)."""
    return np.ascontiguousarray(a, np.float32).reshape(-1, cols)


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _T(T):
    T = np.ascontiguousarray(T, dtype=np.float32).reshape(3, 4)
    return T


def identity():
    return np.hstack([np.eye(3, dtype=np.float32), np.zeros((3, 1), np.float32)])


def rbf_coeff(sigma):
    """RBFKernelWeightEvaluator's coefficient in float: coeff_ = -(WeightT)(0.5) / (sigma * sigma)."""
    sg = np.float32(sigma)
    return float(np.float32(-0.5) / (sg * sg))


def _icp_params(metric, max_iter, tol, max_d2, w_pt, w_pl, max_opt_iter, opt_tol, T_init, pt_rbf_sigma, pl_rbf_sigma,
                **engine):
    """The IcpParams of one ICP run (accum_double and parallel left 0); engine = _engine_fields' keywords."""
    prm = IcpParams()
    _engine_fields(prm, **engine)
    prm.metric = 0 if metric == "p2p" else 1
    prm.max_iter, prm.tol, prm.max_d2 = int(max_iter), tol, max_d2
    prm.w_pt, prm.w_pl = w_pt, w_pl
    prm.max_opt_iter, prm.opt_tol = int(max_opt_iter), opt_tol
    if pt_rbf_sigma is not None:
        prm.pt_weight_kind, prm.pt_weight_coeff = 1, rbf_coeff(pt_rbf_sigma)
    if pl_rbf_sigma is not None:
        prm.pl_weight_kind, prm.pl_weight_coeff = 1, rbf_coeff(pl_rbf_sigma)
    Ti = identity() if T_init is None else _T(T_init)
    for i, v in enumerate(Ti.reshape(-1)):
        prm.T_init[i] = float(v)
    return prm


def num_threads():
    return lib().orc_num_threads()


def set_num_threads(n):
    lib().orc_set_num_threads(C.c_int(n))


# ------------------------------------------------------------------------------------------
# kNN back ends (both satisfy orc_knn_fn)
# ------------------------------------------------------------------------------------------
class BruteKnn:
    """Brute-force restatement of the radius-bounded 1-NN (lowest index wins exact ties)."""

    kind = "port"

    def __init__(self, ref_pts):
        self.pts = _f32(ref_pts)
        self.ctx = BruteCtx(_p(self.pts), self.pts.shape[0])
        self.fn = C.cast(lib().orc_knn1_brute_cb, C.c_void_p)
        self.user = C.cast(C.pointer(self.ctx), C.c_void_p)

    def query(self, qry, max_d2):
        qry = _f32(qry)
        idx = np.empty(qry.shape[0], np.int64)
        d2 = np.empty(qry.shape[0], np.float32)
        lib().orc_knn1_brute(_p(self.pts), C.c_size_t(self.pts.shape[0]), _p(qry), C.c_size_t(qry.shape[0]),
                             C.c_float(max_d2), _p(idx), _p(d2))
        return idx, d2

    def neighborhoods(self, qry, k, r2, stride=None):
        """k nearest with d2 < r2 (k == 0: all within r2), ascending (d2, index): idx [nq, stride], d2, cnt."""
        qry = _f32(qry)
        stride = int(stride or k)
        idx = np.empty((qry.shape[0], stride), np.int64)
        d2 = np.empty((qry.shape[0], stride), np.float32)
        cnt = np.empty(qry.shape[0], np.uint32)
        lib().orc_neighborhoods_brute(_p(self.pts), C.c_size_t(self.pts.shape[0]), _p(qry), C.c_size_t(qry.shape[0]),
                                      C.c_size_t(k), C.c_float(r2), C.c_size_t(stride), _p(idx), _p(d2), _p(cnt))
        return idx, d2, cnt


class RefKnn:
    """The reference's own nanoflann kd-tree (leaf 10, 1 build thread), via oracle/_ref."""

    kind = "reference"

    def __init__(self, ref_pts, max_leaf=10):
        r = ref()
        if r is None:
            raise RuntimeError("oracle/_ref/libcilantro_ref_knn.so not built (needs the reference checkout)")
        self.pts = _f32(ref_pts)
        self.h = C.c_void_p(r.ref_tree_build(_p(self.pts), C.c_size_t(self.pts.shape[0]), C.c_size_t(max_leaf)))
        self.fn = C.cast(r.ref_knn1_radius_cb, C.c_void_p)
        self.user = self.h

    def __del__(self):
        try:
            if self.h:
                ref().ref_tree_free(self.h)
                self.h = None
        except Exception:
            pass

    def query(self, qry, max_d2):
        qry = _f32(qry)
        idx = np.empty(qry.shape[0], np.int64)
        d2 = np.empty(qry.shape[0], np.float32)
        ref().ref_knn1_radius_cb(self.h, _p(qry), C.c_size_t(qry.shape[0]), C.c_float(max_d2), _p(idx), _p(d2))
        return idx, d2

    def nn(self, qry):
        qry = _f32(qry)
        idx = np.empty(qry.shape[0], np.int64)
        d2 = np.empty(qry.shape[0], np.float32)
        ref().ref_nn1(self.h, _p(qry), C.c_size_t(qry.shape[0]), _p(idx), _p(d2))
        return idx, d2

    def knn_in_radius(self, q, k, r2):
        q = np.ascontiguousarray(q, np.float32).reshape(3)
        idx = np.empty(k, np.uint64)
        d2 = np.empty(k, np.float32)
        n = ref().ref_knn_in_radius(self.h, _p(q), C.c_size_t(k), C.c_float(r2), _p(idx), _p(d2))
        return idx[:n].astype(np.int64), d2[:n]

    def neighborhoods(self, qry, k, r2, stride=None):
        """Batched kNNInRadiusSearch (k > 0) or radiusSearch (k == 0): idx [nq, stride], d2, cnt."""
        qry = _f32(qry)
        stride = int(stride or k)
        idx = np.empty((qry.shape[0], stride), np.int64)
        d2 = np.empty((qry.shape[0], stride), np.float32)
        cnt = np.empty(qry.shape[0], np.uint32)
        if k > 0:
            assert stride == k
            ref().ref_knn_in_radius_batch(self.h, _p(qry), C.c_size_t(qry.shape[0]), C.c_size_t(k), C.c_float(r2),
                                          _p(idx), _p(d2), _p(cnt))
        else:
            ref().ref_radius_batch(self.h, _p(qry), C.c_size_t(qry.shape[0]), C.c_float(r2), C.c_size_t(stride),
                                   _p(idx), _p(d2), _p(cnt))
        return idx, d2, cnt


def make_knn(ref_pts, prefer_ref=True):
    if prefer_ref and have_ref():
        return RefKnn(ref_pts)
    return BruteKnn(ref_pts)


# ------------------------------------------------------------------------------------------
# Restated functions
# ------------------------------------------------------------------------------------------
def transform_points(T, pts):
    pts = _f32(pts)
    out = np.empty_like(pts)
    lib().orc_transform_points(_p(_T(T)), _p(pts), C.c_size_t(pts.shape[0]), _p(out))
    return out


def find_correspondences(T, src, knn, max_d2):
    src = _f32(src)
    n = src.shape[0]
    i1 = np.empty(n, np.uint64)
    i2 = np.empty(n, np.uint64)
    v = np.empty(n, np.float32)
    c = lib().orc_find_correspondences(_p(_T(T)), _p(src), C.c_size_t(n), C.c_size_t(knn.pts.shape[0]),
                                       C.c_float(max_d2), knn.fn, knn.user, _p(i1), _p(i2), _p(v))
    return i1[:c].astype(np.int64), i2[:c].astype(np.int64), v[:c]


def kabsch(dst, src, accum_double=False):
    dst, src = _f32(dst), _f32(src)
    assert dst.shape == src.shape
    T = np.empty((3, 4), np.float32)
    ok = lib().orc_kabsch(_p(dst), _p(src), C.c_size_t(dst.shape[0]), C.c_int(int(accum_double)), _p(T))
    return T, bool(ok)


def rotation(L):
    L = np.ascontiguousarray(L, np.float32).reshape(3, 3)
    out = np.empty((3, 3), np.float32)
    lib().orc_rotation(_p(L), _p(out))
    return out


def estimate_combined(dst_p, dst_n, src_p, idx_first, idx_second, w_pt, w_pl, max_iter=1, tol=1e-5,
                      dst_mean=None, src_mean=None, src_n=None, accum_double=False):
    dst_p, dst_n, src_p = _f32(dst_p), _f32(dst_n), _f32(src_p)
    src_n = _f32(src_n) if src_n is not None else None
    i1 = np.ascontiguousarray(idx_first, np.uint64)
    i2 = np.ascontiguousarray(idx_second, np.uint64)
    dm = np.zeros(3, np.float32) if dst_mean is None else np.ascontiguousarray(dst_mean, np.float32)
    sm = np.zeros(3, np.float32) if src_mean is None else np.ascontiguousarray(src_mean, np.float32)
    T = np.empty((3, 4), np.float32)
    ok = lib().orc_estimate_combined(_p(dst_p), _p(dst_n), C.c_size_t(dst_p.shape[0]), _p(src_p), _p(src_n),
                                     _p(i1), _p(i2), C.c_size_t(i1.shape[0]), C.c_float(w_pt), C.c_float(w_pl),
                                     C.c_size_t(max_iter), C.c_float(tol), _p(dm), _p(sm),
                                     C.c_int(int(accum_double)), _p(T))
    return T, bool(ok)


def icp(dst_p, src_p, knn, metric="p2p", dst_n=None, src_n=None, max_iter=15, tol=1e-5, max_d2=1e-4,
        w_pt=0.0, w_pl=1.0, max_opt_iter=1, opt_tol=1e-5, T_init=None, accum_double=False, parallel=False,
        log=False, search_dir="second_to_first", inlier_fraction=1.0, require_reciprocal=False, one_to_one=False,
        f2s_reference=False, pt_rbf_sigma=None, pl_rbf_sigma=None):
    """icp_base.hpp:68-87 driving the p2p or combined/symmetric estimator. Returns a dict.
    pt_rbf_sigma / pl_rbf_sigma: RBFKernelWeightEvaluator<float, float, true>(sigma) as the point-to-point /
    point-to-plane correspondence weight evaluator (common_pair_evaluators.hpp:46-79); None = UnityWeightEvaluator."""
    dst_p, src_p = _f32(dst_p), _f32(src_p)
    dst_n = _f32(dst_n) if dst_n is not None else None
    src_n = _f32(src_n) if src_n is not None else None
    prm = _icp_params(metric, max_iter, tol, max_d2, w_pt, w_pl, max_opt_iter, opt_tol, T_init, pt_rbf_sigma,
                      pl_rbf_sigma, search_dir=search_dir, inlier_fraction=inlier_fraction,
                      require_reciprocal=require_reciprocal, one_to_one=one_to_one, f2s_reference=f2s_reference)
    prm.accum_double = int(accum_double)
    prm.parallel = int(parallel)
    res = IcpResult()
    tlog = np.zeros((max(int(max_iter), 1), 3, 4), np.float32) if log else None
    if prm.metric == 1:
        assert dst_n is not None
    lib().orc_icp(_p(dst_p), _p(dst_n), C.c_size_t(dst_p.shape[0]), _p(src_p), _p(src_n),
                  C.c_size_t(src_p.shape[0]), C.byref(prm), knn.fn, knn.user, C.byref(res), _p(tlog))
    out = {
        "T": np.array(list(res.T), np.float32).reshape(3, 4),
        "iterations": int(res.iterations),
        "last_delta": float(res.last_delta),
        "converged": bool(res.converged),
        "num_corr": int(res.last_num_corr),
        "t_knn_s": float(res.t_knn_s),
        "t_est_s": float(res.t_est_s),
    }
    if log:
        out["T_log"] = tlog[: res.iterations]
    return out


def _engine_fields(prm, search_dir, inlier_fraction, require_reciprocal, one_to_one, f2s_reference=False):
    prm.search_dir = SEARCH_DIR[search_dir] if isinstance(search_dir, str) else int(search_dir)
    prm.inlier_fraction = float(inlier_fraction)
    prm.require_reciprocal = int(require_reciprocal)
    prm.one_to_one = int(one_to_one)
    # FIRST_TO_SECOND searches: brute force (lowest index on exact ties, the CUDA path's rule) or, on request, the
    # reference's own nanoflann with the tree over the transformed source rebuilt per call (ties: traversal order)
    prm.f2s_fn = C.cast(ref().ref_knn1_build_query, C.c_void_p) if (f2s_reference and have_ref()) else None


def engine_correspondences(dst_p, src_p, T, knn, max_d2, search_dir="second_to_first", inlier_fraction=1.0,
                           require_reciprocal=False, one_to_one=False, f2s_reference=False):
    """CorrespondenceSearchKDTree::findCorrespondences(T).getCorrespondences(): (first, second, value)."""
    dst_p, src_p = _f32(dst_p), _f32(src_p)
    prm = IcpParams()
    prm.max_d2 = max_d2
    _engine_fields(prm, search_dir, inlier_fraction, require_reciprocal, one_to_one, f2s_reference)
    cap = dst_p.shape[0] + src_p.shape[0]
    i1 = np.empty(cap, np.uint64)
    i2 = np.empty(cap, np.uint64)
    v = np.empty(cap, np.float32)
    m = lib().orc_engine_correspondences(_p(dst_p), C.c_size_t(dst_p.shape[0]), _p(src_p), C.c_size_t(src_p.shape[0]),
                                         _p(_T(T)), C.byref(prm), knn.fn, knn.user, _p(i1), _p(i2), _p(v))
    return i1[:m].astype(np.int64), i2[:m].astype(np.int64), v[:m].copy()


def icp_residuals(dst_p, src_p, T, knn, metric="p2p", dst_n=None, src_n=None, w_pt=0.0, w_pl=1.0):
    dst_p, src_p = _f32(dst_p), _f32(src_p)
    dst_n = _f32(dst_n) if dst_n is not None else None
    src_n = _f32(src_n) if src_n is not None else None
    res = np.empty(src_p.shape[0], np.float32)
    lib().orc_icp_residuals(_p(dst_p), _p(dst_n), C.c_size_t(dst_p.shape[0]), _p(src_p), _p(src_n),
                            C.c_size_t(src_p.shape[0]), _p(_T(T)), C.c_int(0 if metric == "p2p" else 1),
                            C.c_float(w_pt), C.c_float(w_pl), knn.fn, knn.user, _p(res))
    return res


def kmeans_assign(pts, cent, labels=None):
    pts, cent = _f32(pts), _f32(cent)
    if labels is None:
        labels = np.zeros(pts.shape[0], np.uint64)
    else:
        labels = np.ascontiguousarray(labels, np.uint64).copy()
    unchanged = lib().orc_kmeans_assign(_p(pts), C.c_size_t(pts.shape[0]), _p(cent), C.c_size_t(cent.shape[0]),
                                        _p(labels))
    return labels, bool(unchanged)


def kmeans_seed_indices(n, k, seed):
    out = np.empty(k, np.uint64)
    lib().orc_kmeans_seed_indices(C.c_size_t(n), C.c_size_t(k), C.c_uint32(seed), _p(out))
    return out.astype(np.int64)


def kmeans(pts, cent0, max_iter=100, tol=float(np.finfo(np.float32).eps)):
    pts = _f32(pts)
    cent = _f32(cent0).copy()
    labels = np.zeros(pts.shape[0], np.uint64)
    it = lib().orc_kmeans(_p(pts), C.c_size_t(pts.shape[0]), _p(cent), C.c_size_t(cent.shape[0]),
                          C.c_size_t(max_iter), C.c_float(tol), _p(labels))
    return cent, labels.astype(np.int64), int(it)


def ransac_score(dst, src, T_h, thresh):
    dst, src = _f32(dst), _f32(src)
    T_h = np.ascontiguousarray(T_h, np.float32).reshape(-1, 3, 4)
    counts = np.empty(T_h.shape[0], np.uint32)
    lib().orc_ransac_score(_p(dst), _p(src), C.c_size_t(dst.shape[0]), _p(T_h), C.c_size_t(T_h.shape[0]),
                           C.c_float(thresh), _p(counts))
    return counts


def ransac_samples(n, sample_size, iters, seed):
    out = np.empty((iters, sample_size), np.uint64)
    lib().orc_ransac_samples(C.c_size_t(n), C.c_size_t(sample_size), C.c_size_t(iters), C.c_uint32(seed), _p(out))
    return out.astype(np.int64)


def ransac_fit_samples(dst, src, samples):
    dst, src = _f32(dst), _f32(src)
    samples = np.ascontiguousarray(samples, np.uint64)
    H, ss = samples.shape
    T_h = np.empty((H, 3, 4), np.float32)
    lib().orc_ransac_fit_samples(_p(dst), _p(src), _p(samples), C.c_size_t(ss), C.c_size_t(H), _p(T_h))
    return T_h


def ransac_rigid(dst, src, seed, max_iter=100, thresh=0.01, inlier_count_thresh=None, re_estimate=True,
                 sample_size=3):
    dst, src = _f32(dst), _f32(src)
    n = dst.shape[0]
    if inlier_count_thresh is None:
        inlier_count_thresh = n // 2 + n % 2  # ransac_transform_estimator.hpp:27
    res = RansacResult()
    inl = np.empty(n, np.uint64)
    resid = np.zeros(n, np.float32)
    lib().orc_ransac_rigid(_p(dst), _p(src), C.c_size_t(n), C.c_uint32(seed), C.c_size_t(sample_size),
                           C.c_size_t(inlier_count_thresh), C.c_size_t(max_iter), C.c_float(thresh),
                           C.c_int(int(re_estimate)), C.byref(res), _p(inl), _p(resid))
    return {
        "T": np.array(list(res.T), np.float32).reshape(3, 4),
        "iterations": int(res.iterations),
        "num_inliers": int(res.num_inliers),
        "best_iteration": int(res.best_iteration),
        "inliers": inl[: res.num_inliers].astype(np.int64),
        "residuals": resid,
    }


def estimate_normals(pts, knn, k=0, radius2=None, view_point=None, ref_normals=None, neighbors=None):
    """NormalEstimation::estimateNormalsAndCurvature{KNN,Radius,KNNInRadius} (core/normal_estimation.hpp:83-232)
    on neighbourhoods from `knn` (RefKnn = the reference's nanoflann), or on precomputed `neighbors` = (idx, cnt).
    Returns normals, curvature, cov6, cnt."""
    pts = _f32(pts)
    n = pts.shape[0]
    r2 = FLT_MAX if radius2 is None else float(radius2)
    if neighbors is not None:
        idx = np.ascontiguousarray(neighbors[0], np.int64)
        cnt = np.ascontiguousarray(neighbors[1], np.uint32)
    elif k > 0:
        idx, _, cnt = knn.neighborhoods(pts, k, r2)
    else:
        _, _, cnt = knn.neighborhoods(pts, 0, r2, stride=1)
        idx, _, cnt = knn.neighborhoods(pts, 0, r2, stride=max(1, int(cnt.max()) if n else 1))
    normals = np.empty((n, 3), np.float32)
    curv = np.empty(n, np.float32)
    cov6 = np.empty((n, 6), np.float32)
    vp = None if view_point is None else np.ascontiguousarray(view_point, np.float32).reshape(3)
    lib().orc_normals_from_neighbors(_p(pts), C.c_size_t(n), _p(idx), C.c_size_t(idx.shape[1]), _p(cnt), _p(vp),
                                     _p(_f32(ref_normals) if ref_normals is not None else None), _p(normals), _p(curv), _p(cov6))
    return normals, curv, cov6, cnt


def grid_downsample(pts, bin_size, normals=None, colors=None, min_points=1, order=0):
    """PointCloud::gridDownsample (serial sums; order 0 = map order, 1 = first occurrence): points, normals, colors."""
    pts = _f32(pts)
    n = pts.shape[0]
    nrm = _f32(normals) if normals is not None else None
    col = _f32(colors) if colors is not None else None
    o_p = np.empty((max(n, 1), 3), np.float32)
    o_n = np.empty((max(n, 1), 3), np.float32) if nrm is not None else None
    o_c = np.empty((max(n, 1), 3), np.float32) if col is not None else None
    m = lib().orc_grid_downsample(_p(pts), _p(nrm), _p(col), C.c_size_t(n), C.c_float(bin_size), C.c_size_t(min_points),
                                  C.c_int(order), _p(o_p), _p(o_n), _p(o_c))
    return o_p[:m].copy(), (o_n[:m].copy() if o_n is not None else None), (o_c[:m].copy() if o_c is not None else None)


def pca(pts, accum_double=False):
    pts = _f32(pts)
    mean = np.empty(3, np.float32)
    cov = np.empty((3, 3), np.float32)
    ev = np.empty(3, np.float32)
    evec = np.empty((3, 3), np.float32)
    ok = lib().orc_pca(_p(pts), C.c_size_t(pts.shape[0]), C.c_int(int(accum_double)), _p(mean), _p(cov), _p(ev),
                       _p(evec))
    return {"ok": bool(ok), "mean": mean, "cov": cov, "eigenvalues": ev, "eigenvectors": evec}
