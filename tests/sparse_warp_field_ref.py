"""A vectorised fp64 statement of estimateSparseWarpFieldCombinedMetric's linear system (registration/
warp_field_estimation.hpp:1486-1805) in the reference's row and column layout, and of resampleTransforms
(warp_field_utilities.hpp:14-48), for the sparse warp-field tests. Independent of the oracle's C++: rotations are
built as Rz(c) Ry(b) Rx(a) and their derivatives in numpy.

At is (6 m unknowns) x (equations): the point-to-point rows (3 per correspondence), then the point-to-plane rows (1
per correspondence), then 6 rows per regularisation arc (N[0], N[j]) in list order. The entry of node n_k in a data
row of source point i is the row's gradient times (sqrt(w) / W_i) w_k; the right-hand side is the residual times
sqrt(w)."""
import numpy as np
import scipy.sparse as sp


def rbf(d2, sigma):
    """RBFKernelWeightEvaluator<float, float, true> with its float coefficient -0.5f / sigma^2, in fp64."""
    sg = np.float32(sigma)
    return np.exp(float(np.float32(-0.5) / (sg * sg)) * np.asarray(d2, np.float64))


def sqrt_huber(x, delta):
    xa = np.abs(x)
    return np.where(xa > delta, np.sqrt(delta * np.maximum(xa - 0.5 * delta, 0.0)), np.sqrt(0.5) * xa)


def sqrt_huber_d(x, delta):
    xa = np.abs(x)
    big = xa > delta
    v = np.where(big, delta / (2.0 * np.sqrt(np.where(big, delta * (xa - 0.5 * delta), 1.0))), np.sqrt(0.5))
    return np.where(x < 0, -v, v)


def _rot(a, b, c):
    """R = Rz(c) Ry(b) Rx(a) and dR/da, dR/db, dR/dc, each (k, 3, 3)."""
    z, o = np.zeros_like(a), np.ones_like(a)
    ca, sa, cb, sb, cc, sc = np.cos(a), np.sin(a), np.cos(b), np.sin(b), np.cos(c), np.sin(c)
    Rx = np.stack([o, z, z, z, ca, -sa, z, sa, ca], -1).reshape(-1, 3, 3)
    Ry = np.stack([cb, z, sb, z, o, z, -sb, z, cb], -1).reshape(-1, 3, 3)
    Rz = np.stack([cc, -sc, z, sc, cc, z, z, z, o], -1).reshape(-1, 3, 3)
    dRx = np.stack([z, z, z, z, -sa, -ca, z, ca, -sa], -1).reshape(-1, 3, 3)
    dRy = np.stack([-sb, z, cb, z, z, z, -cb, z, -sb], -1).reshape(-1, 3, 3)
    dRz = np.stack([-sc, -cc, z, cc, -sc, z, z, z, z], -1).reshape(-1, 3, 3)
    return Rz @ Ry @ Rx, Rz @ Ry @ dRx, Rz @ dRy @ Rx, dRz @ Ry @ Rx


def sorted_lists(ctrl, sigma):
    """Per entry of the control CSR, sorted stably by node within each list: (point, node, weight) and W per point
    (summed over the list)."""
    off, idx, d2 = (np.asarray(a) for a in ctrl)
    n = off.shape[0] - 1
    pt = np.repeat(np.arange(n), np.diff(off).astype(np.int64))
    w = rbf(d2, sigma)
    W = np.bincount(pt, weights=w, minlength=n)
    order = np.lexsort((np.arange(pt.shape[0]), idx, pt))
    return pt[order], np.asarray(idx, np.int64)[order], w[order], W


def system(dst, nrm, src, first, second, ctrl, m, reg, x, w_pt, w_pl, stiffness, huber, reg_sigma, ctrl_sigma):
    """(At, b): At a scipy CSR of (6 m) x equations, b the right-hand side, at the node unknowns x (m, 6)."""
    dst, src = np.asarray(dst, np.float64), np.asarray(src, np.float64)
    w_pt, w_pl, stiffness, huber = (float(np.float32(v)) for v in (w_pt, w_pl, stiffness, huber))  # float parameters
    x = np.asarray(x, np.float64).reshape(m, 6)
    first, second = np.asarray(first, np.int64), np.asarray(second, np.int64)
    pt, node, w, W = sorted_lists(ctrl, ctrl_sigma)
    n = src.shape[0]
    xbar = np.zeros((n, 6))
    np.add.at(xbar, pt, w[:, None] * x[node])
    safe = np.where(W != 0, W, 1.0)
    xbar = np.where((W != 0)[:, None], xbar / safe[:, None], 0.0)
    R, Da, Db, Dc = _rot(xbar[:, 0], xbar[:, 1], xbar[:, 2])
    start = np.searchsorted(pt, np.arange(n + 1))  # the sorted list of point i: start[i] .. start[i+1]-1

    rows, cols, vals, rhs = [], [], [], []
    eq = 0

    def data_block(grads, res, cw):
        """grads (c, r, 6): the per-correspondence rows' gradients; res (c, r); cw the correspondence weight."""
        nonlocal eq
        c, r = res.shape
        i = second
        scale = np.where(W[i] != 0, cw / safe[i], 0.0)
        cws = np.where(W[i] != 0, cw, 0.0)
        for k in range(c):
            lo, hi = start[i[k]], start[i[k] + 1]
            for rr in range(r):
                for t in range(lo, hi):
                    rows.extend([eq + k * r + rr] * 6)
                    cols.extend(6 * node[t] + np.arange(6))
                    vals.extend(grads[k, rr] * scale[k] * w[t])
        rhs.append((res * cws[:, None]).ravel())
        eq += c * r

    s = src[second]
    d = dst[first]
    das = np.einsum("kij,kj->ki", Da[second], s)
    dbs = np.einsum("kij,kj->ki", Db[second], s)
    dcs = np.einsum("kij,kj->ki", Dc[second], s)
    ts = d - (np.einsum("kij,kj->ki", R[second], s) + xbar[second, 3:])
    c = second.shape[0]
    if c and w_pt > 0:
        g = np.zeros((c, 3, 6))
        g[:, :, 0], g[:, :, 1], g[:, :, 2] = das, dbs, dcs
        g[:, [0, 1, 2], [3, 4, 5]] = 1.0
        data_block(g, ts, np.sqrt(w_pt))
    if c and w_pl > 0:
        nn = np.asarray(nrm, np.float64)[first]
        g = np.stack([(nn * das).sum(1), (nn * dbs).sum(1), (nn * dcs).sum(1), nn[:, 0], nn[:, 1], nn[:, 2]], 1)
        data_block(g[:, None, :], (nn * ts).sum(1)[:, None], np.sqrt(w_pl))
    roff, ridx, rd2 = (np.asarray(a) for a in reg)
    for j in range(roff.shape[0] - 1):
        nb = ridx[roff[j]:roff[j + 1]]
        for t in range(1, nb.shape[0]):
            so, no = sorted((int(nb[0]), int(nb[t])))
            wt = np.sqrt(stiffness) * np.sqrt(rbf(rd2[roff[j] + t], reg_sigma))
            diff = x[so] - x[no]
            h = wt * sqrt_huber_d(diff, huber)
            for u in range(6):
                rows.extend([eq + u, eq + u])
                cols.extend([6 * so + u, 6 * no + u])
                vals.extend([h[u], -h[u]])
            rhs.append(-wt * sqrt_huber(diff, huber))
            eq += 6
    A = sp.csr_matrix((np.asarray(vals, np.float64), (np.asarray(rows), np.asarray(cols))), shape=(eq, 6 * m))
    return A.T.tocsr(), (np.concatenate(rhs) if rhs else np.zeros(0))


def resample(T, ctrl, sigma):
    """resampleTransforms in fp64: the weighted blend over each list in its order, then the nearest rotation (SVD,
    a reflection repaired on the largest singular value)."""
    off, idx, d2 = (np.asarray(a) for a in ctrl)
    T = np.asarray(T, np.float64).reshape(-1, 3, 4)
    n = off.shape[0] - 1
    pt = np.repeat(np.arange(n), np.diff(off).astype(np.int64))
    w = rbf(d2, sigma)
    L = np.zeros((n, 3, 4))
    np.add.at(L, pt, w[:, None, None] * T[np.asarray(idx, np.int64)])
    W = np.bincount(pt, weights=w, minlength=n)
    out = np.tile(np.hstack([np.eye(3), np.zeros((3, 1))]), (n, 1, 1))
    ok = W != 0
    L = L[ok] / W[ok, None, None]
    U, _, Vt = np.linalg.svd(L[:, :, :3])
    # LinearTransform::rotation() (space_transformations.hpp:43-51) repairs a reflection on column 0 of U: the largest
    # singular value's, as numpy's and Eigen's SVDs sort them descending
    D = np.ones((L.shape[0], 3))
    D[:, 0] = np.sign(np.linalg.det(U @ Vt))
    out[ok, :, :3] = (U * D[:, None, :]) @ Vt
    out[ok, :, 3] = L[:, :, 3]
    return out


def make_case(n, res, seed=1, k_ctrl=4, k_reg=8, spacing=0.005):
    """The reference example's sparse recipe on synth.warp_pair: nodes = grid-downsampled source at `res`, 4-NN
    control lists, 8-NN node neighbourhoods. Returns dict(dst, dst_normals, src, nodes, ctrl, reg, m)."""
    import oracle
    from cilantro_b200 import capi, synth

    P = synth.warp_pair(n, seed=seed, spacing=spacing)
    nodes, _, _ = oracle.grid_downsample(P["src"], res)
    knn = oracle.BruteKnn(nodes)
    P["nodes"] = nodes
    P["m"] = nodes.shape[0]
    P["ctrl"] = capi.neighborhood_csr(*knn.neighborhoods(P["src"], k_ctrl, 3.0e38))
    P["reg"] = capi.neighborhood_csr(*knn.neighborhoods(nodes, k_reg, 3.0e38))
    return P
