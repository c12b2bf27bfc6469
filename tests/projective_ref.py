"""numpy fp32 restatement of the projective correspondence search of rigid ICP (DESIGN §4.21,
CorrespondenceSearchProjective::find_correspondences_): the index map of depth_images_ref over the destination, then per
source point p = T s (icp_ref.apply_f32), its pixel (depth_images_ref._project), the map's point and the contract
distance ((dx dx + dy dy) + dz dz, d = p - dst), kept iff < max_d2, in ascending source index; with 0 < fraction < 1
the stable sort on the value keeps the first llround(fraction m) pairs (filterCorrespondencesFraction, ties in list
order). On top, a float64 ICP loop whose correspondences come from this search at each fp32 iterate."""
import numpy as np

import depth_images_ref as dimg
import icp_ref

F = np.float32
EMPTY = np.iinfo(np.uint64).max


def correspondences(dst, src, T, K, w, h, extrinsics=None, max_d2=F(1e-4), fraction=1.0):
    """(first = destination index, second = source index, value) of the projective search at transform T."""
    src = np.asarray(src, F).reshape(-1, 3)
    none = (np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, F))
    if w == 0 or h == 0 or src.shape[0] == 0 or np.asarray(dst).shape[0] == 0:
        return none
    imap = dimg.points_to_index_map(dst, K, w, h, extrinsics).reshape(-1)
    q = icp_ref.apply_f32(T, src)
    _, pix = dimg._project(q, K, extrinsics, w, h)
    second = np.nonzero(pix >= 0)[0]
    ind = imap[pix[second]]
    hit = ind != EMPTY
    second, first = second[hit], ind[hit].astype(np.int64)
    p = np.asarray(dst, F)[first]
    with np.errstate(all="ignore"):
        d = q[second] - p
        value = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    keep = value < F(max_d2)
    first, second, value = first[keep], second[keep], value[keep].astype(F)
    if 0.0 < fraction < 1.0 and first.size:
        order = np.argsort(value, kind="stable")
        m = int(np.floor(np.float64(fraction) * first.size + 0.5))  # llround of a non-negative value
        order = order[:m]
        first, second, value = first[order], second[order], value[order]
    return first, second, value


def icp_loop(dst, src, K, w, h, extrinsics, T0, max_iter, max_d2, metric="p2p", dst_n=None, src_n=None, w_pt=0.0,
             w_pl=1.0):
    """max_iter iterations (no convergence test) of icp_ref's float64 steps over the projective correspondences at
    each iterate rounded to fp32: returns T."""
    dst = np.asarray(dst, F)
    src = np.asarray(src, F)
    T = np.asarray(T0, np.float64)
    fin_d, fin_s = icp_ref.finite_rows(dst), icp_ref.finite_rows(src)
    dm = dst[fin_d].astype(np.float64).mean(0).astype(F)
    sm = src[fin_s].astype(np.float64).mean(0).astype(F)
    for _ in range(max_iter):
        Tf = T.astype(F)
        first, second, _ = correspondences(dst, src, Tf, K, w, h, extrinsics, max_d2)
        if metric == "p2p":
            Tn, _ = icp_ref.p2p_step(dst, src, Tf, first, second)
        else:
            Tn, _ = icp_ref.combined_step(dst, dst_n, src, Tf, first, second, w_pt, w_pl, dm, sm, src_n)
        T = Tn
    return T
