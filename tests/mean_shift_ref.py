"""An independent numpy / scipy statement of MeanShift3f::cluster (clustering/mean_shift.hpp:37-115) for small
inputs: cKDTree.query_ball_point for the candidates, the fp32 distance ((dx^2 + dy^2) + dz^2) < r2 as the test,
lists sorted on (d2, index), sequential fp32 sums with np.add.accumulate, and the greedy clustering in Python."""
import numpy as np
from scipy.spatial import cKDTree

F = np.float32


def _d2(q, p):
    d = (q[None, :] - p).astype(F)
    return ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(F)


def _seq_sum(v):
    """0 + v[0] + v[1] + ... in fp32, in order."""
    return np.add.accumulate(np.concatenate([np.zeros(1, F), np.asarray(v, F)]), dtype=F)[-1]


def mean_shift(pts, kernel_radius, max_iter, cluster_tol, convergence_tol=float(np.finfo(F).eps), seeds=None,
               rbf_sigma=None):
    pts = np.asarray(pts, F).reshape(-1, 3)
    s = (pts if seeds is None else np.asarray(seeds, F).reshape(-1, 3)).copy()
    r2 = F(kernel_radius) * F(kernel_radius)
    tol2 = F(convergence_tol) * F(convergence_tol)
    coeff = None if rbf_sigma is None else F(-0.5) / (F(rbf_sigma) * F(rbf_sigma))
    finite = np.isfinite(pts).all(axis=1)
    tree = cKDTree(pts[finite].astype(np.float64)) if finite.any() else None
    fidx = np.flatnonzero(finite)
    conv = np.zeros(s.shape[0], bool)
    it = 0
    while it < max_iter:
        all_conv = True
        for i in range(s.shape[0]):
            if conv[i]:
                continue
            q = s[i]
            cand = np.zeros(0, np.int64)
            if tree is not None and np.isfinite(q).all() and r2 > 0:
                cand = fidx[np.asarray(tree.query_ball_point(q.astype(np.float64), float(np.sqrt(r2)) * 1.001 + 1e-30),
                                       np.int64)]
            d2 = _d2(q, pts[cand]) if cand.size else np.zeros(0, F)
            keep = d2 < r2
            cand, d2 = cand[keep], d2[keep]
            o = np.lexsort((cand, d2))
            cand, d2 = cand[o], d2[o]
            w = np.ones(cand.size, F) if coeff is None else np.exp(coeff * d2).astype(F)
            with np.errstate(divide="ignore", invalid="ignore"):
                acc = np.array([_seq_sum(w * pts[cand, c]) for c in range(3)], F)
                inv = F(1.0) / _seq_sum(w)
                m = (acc * inv).astype(F)
                dd = (q - m).astype(F)
                sq = (dd[0] * dd[0] + dd[1] * dd[1]) + dd[2] * dd[2]
            if sq < tol2:
                conv[i] = True
            else:
                all_conv = False
            s[i] = m
        it += 1
        if all_conv:
            break
    # greedy clustering
    ct2 = F(cluster_tol) * F(cluster_tol)
    clusters = []
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(s.shape[0]):
            for c in clusters:
                dd = (s[i] - s[c[0]]).astype(F)
                if (dd[0] * dd[0] + dd[1] * dd[1]) + dd[2] * dd[2] < ct2:
                    c.append(i)
                    break
            else:
                clusters.append([i])
        modes = np.array([[_seq_sum(s[c, k]) * (F(1.0) / F(len(c))) for k in range(3)] for c in clusters], F)
    p2c = np.zeros(s.shape[0], np.int64)
    for ci, c in enumerate(clusters):
        p2c[c] = ci
    off = np.concatenate([[0], np.cumsum([len(c) for c in clusters])]).astype(np.int64)
    members = np.array([i for c in clusters for i in c], np.int64)
    return {"offsets": off, "points": members, "point_to_cluster": p2c, "num_clusters": len(clusters),
            "shifted_seeds": s, "modes": modes.reshape(-1, 3), "iterations": it}
