"""Seeded synthetic workloads (SURVEY.md §8(d)); shared by tests/ and bench.py. numpy only."""
import numpy as np


def rigid_from_axis_angle(axis, angle, t):
    axis = np.asarray(axis, np.float64)
    axis = axis / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    R = np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * (K @ K)
    T = np.zeros((3, 4), np.float64)
    T[:, :3] = R
    T[:, 3] = np.asarray(t, np.float64)
    return T


def invert(T):
    T = np.asarray(T, np.float64)
    R, t = T[:, :3], T[:, 3]
    out = np.zeros((3, 4), np.float64)
    out[:, :3] = R.T
    out[:, 3] = -R.T @ t
    return out


def apply(T, pts):
    T = np.asarray(T, np.float64)
    return (np.asarray(pts, np.float64) @ T[:, :3].T + T[:, 3]).astype(np.float32)


def t_ref_default():
    """AngleAxis(0.02 rad about (1,1,1)/sqrt(3)), t = (0.01, -0.005, 0.008)."""
    return rigid_from_axis_angle([1, 1, 1], 0.02, [0.01, -0.005, 0.008])


def t_ref_for(n):
    """Generating pose for an n-point uniform cloud in the unit cube.

    SURVEY.md §8(d) proposes AngleAxis(0.02 rad, (1,1,1)/sqrt 3), t = (0.01,-0.005,0.008) for every
    size. Measured here with the oracle: at 1 M points (mean spacing 0.01) that offset (up to 0.03 at
    the cube corners) is outside ICP's basin of convergence on a dense uniform cloud — nearest
    neighbours are almost all wrong matches and BOTH the reference path and ours stall at
    |T - T_ref|_F = 3e-2. The work per iteration is unchanged, but the run is useless as a
    correctness check, so the pose is scaled with the point spacing s = n^(-1/3): angle =
    min(0.02, s/4), translation scaled by the same factor. For n <= 2000 this is SURVEY's pose."""
    s = float(n) ** (-1.0 / 3.0)
    f = min(1.0, (s / 4.0) / 0.02)
    return rigid_from_axis_angle([1, 1, 1], 0.02 * f, [0.01 * f, -0.005 * f, 0.008 * f])


def icp_pair(n, seed=1, noise=0.001, with_normals=False, n_src=None, T_ref=None):
    """dst uniform in [0,1)^3; src = T_ref^-1 dst + uniform noise in +-noise (SURVEY §8(d) configs 2/3).

    Returns dst (n,3), src (n_src,3), dst_normals or None, T_ref (3,4 float64): the transform ICP
    should recover (src -> dst)."""
    rng = np.random.default_rng(seed)
    dst = rng.random((n, 3), dtype=np.float32)
    if T_ref is None:
        T_ref = t_ref_for(n)
    m = n if n_src is None else n_src
    base = dst[:m] if m <= n else rng.random((m, 3), dtype=np.float32)
    src = apply(invert(T_ref), base)
    src = (src + (rng.random((m, 3), dtype=np.float32) - 0.5) * np.float32(2 * noise)).astype(np.float32)
    nrm = None
    if with_normals:
        g = rng.standard_normal((n, 3)).astype(np.float32)
        nrm = (g / np.linalg.norm(g, axis=1, keepdims=True)).astype(np.float32)
    return dst, src, nrm, T_ref


def surface_cloud(n, seed=1, noise=0.0005):
    """A scanned-surface stand-in: the sheet z = 0.5 + 0.1 sin(6x) cos(5y) over [0,1)^2, sampled uniformly in
    (x, y) with Gaussian noise along z. Returns points (n,3) float32 and the analytic unit normals (n,3), +z side."""
    rng = np.random.default_rng(seed)
    xy = rng.random((n, 2))
    x, y = xy[:, 0], xy[:, 1]
    z = 0.5 + 0.1 * np.sin(6 * x) * np.cos(5 * y) + noise * rng.standard_normal(n)
    g = np.stack([-0.6 * np.cos(6 * x) * np.cos(5 * y), 0.5 * np.sin(6 * x) * np.sin(5 * y), np.ones(n)], axis=1)
    g /= np.linalg.norm(g, axis=1, keepdims=True)
    return np.stack([x, y, z], axis=1).astype(np.float32), g.astype(np.float32)


def rigid_icp_example_pair(points, normals, seed=1):
    """The input recipe of the reference's examples/rigid_icp.cpp:25-65 on a loaded scan (BASELINE config 1):
    src = dst + 0.01 * U(-1,1)^3 (normals + 0.02 * U, re-normalised), dst keeps only x > -0.4, then
    src <- tf_ref * src with tf_ref = Rz(-0.1) Ry(0.1) Rx(-0.1), t = (-0.20, -0.05, 0.10).
    Returns dst_p, dst_n, src_p, src_n, tf_ref (3x4 float64); ICP should recover tf_ref^-1."""
    rng = np.random.default_rng(seed)
    p = np.asarray(points, np.float32)
    n = np.asarray(normals, np.float32)
    src_p = (p + np.float32(0.01) * (rng.random(p.shape, dtype=np.float32) * 2 - 1)).astype(np.float32)
    src_n = n + np.float32(0.02) * (rng.random(n.shape, dtype=np.float32) * 2 - 1)
    src_n = (src_n / np.linalg.norm(src_n, axis=1, keepdims=True)).astype(np.float32)
    keep = p[:, 0] > np.float32(-0.4)
    dst_p, dst_n = np.ascontiguousarray(p[keep]), np.ascontiguousarray(n[keep])

    def rot(axis, a):
        return np.asarray(rigid_from_axis_angle(axis, a, [0, 0, 0]))[:, :3]

    R = rot([0, 0, 1], -0.1) @ rot([0, 1, 0], 0.1) @ rot([1, 0, 0], -0.1)
    tf_ref = np.hstack([R, np.array([[-0.20], [-0.05], [0.10]])])
    src_p = apply(tf_ref, src_p).astype(np.float32)
    src_n = (src_n.astype(np.float64) @ R.T).astype(np.float32)
    return dst_p, dst_n, src_p, src_n, tf_ref


def kmeans_data(n, k, seed=1):
    """uniform [0,1)^3 points; initial centroids = first k points of a seeded shuffle (config 4)."""
    rng = np.random.default_rng(seed)
    pts = rng.random((n, 3), dtype=np.float32)
    idx = rng.permutation(n)[:k]
    return pts, pts[idx].copy()


def ransac_pairs(n, inlier_frac=0.3, seed=1, sigma=0.002):
    """src uniform [0,1)^3; dst = T_ref src + N(0, sigma^2) for inliers, uniform otherwise (config 5)."""
    rng = np.random.default_rng(seed)
    src = rng.random((n, 3), dtype=np.float32)
    T_ref = t_ref_default()
    dst = apply(T_ref, src) + (rng.standard_normal((n, 3)) * sigma).astype(np.float32)
    out = rng.random(n) >= inlier_frac
    dst[out] = rng.random((int(out.sum()), 3), dtype=np.float32)
    return dst.astype(np.float32), src, T_ref, ~out


def frobenius(Ta, Tb):
    return float(np.linalg.norm(np.asarray(Ta, np.float64) - np.asarray(Tb, np.float64)))


def segment_scene(n, seed=1):
    """A floor and separated boxes and plates, sampled on cell-centred lattices of spacing ~h with analytic
    (axis-aligned, exact) normals, in random point order. Objects are >= 0.1 apart, so for a radius r with
    h < r < 0.1 (and r > 0.71 h, the gap across a box edge):
      - AlwaysTrueEvaluator: one component per object (floor, each box, each plate);
      - NormalsProximityEvaluator with a small angle: one component per planar face (6 per box).
    Returns dict(points, normals, face (component id per point under the angle test), object (id under
    AlwaysTrue), spacing h, faces (number of faces), objects (number of objects))."""
    rng = np.random.default_rng(seed)
    boxes = [(0.2, 0.2), (0.6, 0.2), (0.2, 0.6)]  # (x, y) centres; side 0.2, z in [0.1, 0.3]
    # (origin, u edge, v edge, normal): floor, a horizontal plate, a vertical plate
    quads = [((0.0, 0.0, 0.0), (1.0, 0, 0), (0, 1.0, 0), (0, 0, 1.0)),
             ((0.55, 0.55, 0.5), (0.3, 0, 0), (0, 0.3, 0), (0, 0, 1.0)),
             ((0.9, 0.1, 0.1), (0, 0.3, 0), (0, 0, 0.3), (1.0, 0, 0))]
    area = 1.0 + 0.09 + 0.09 + len(boxes) * 6 * 0.04
    h = float(np.sqrt(area / n))
    faces = []  # (origin, u, v, normal, object id)
    for o, (u, v, nrm) in enumerate((q[1:] for q in quads)):
        faces.append((quads[o][0], u, v, nrm, o))
    for b, (cx, cy) in enumerate(boxes):
        x0, y0, z0, s = cx - 0.1, cy - 0.1, 0.1, 0.2
        obj = len(quads) + b
        faces += [((x0, y0, z0), (s, 0, 0), (0, s, 0), (0, 0, -1.0), obj), ((x0, y0, z0 + s), (s, 0, 0), (0, s, 0), (0, 0, 1.0), obj),
                  ((x0, y0, z0), (s, 0, 0), (0, 0, s), (0, -1.0, 0), obj), ((x0, y0 + s, z0), (s, 0, 0), (0, 0, s), (0, 1.0, 0), obj),
                  ((x0, y0, z0), (0, s, 0), (0, 0, s), (-1.0, 0, 0), obj), ((x0 + s, y0, z0), (0, s, 0), (0, 0, s), (1.0, 0, 0), obj)]
    pts, nrms, face_id, obj_id = [], [], [], []
    for f, (org, u, v, nrm, obj) in enumerate(faces):
        u, v = np.asarray(u), np.asarray(v)
        qu = max(1, int(round(np.linalg.norm(u) / h)))
        qv = max(1, int(round(np.linalg.norm(v) / h)))
        a, b = np.meshgrid((np.arange(qu) + 0.5) / qu, (np.arange(qv) + 0.5) / qv, indexing="ij")
        a, b = a.ravel(), b.ravel()
        # in-plane jitter of +-5 % of the spacing (the normal direction stays exact)
        a = a + rng.uniform(-0.05, 0.05, a.shape) / qu
        b = b + rng.uniform(-0.05, 0.05, b.shape) / qv
        pts.append(np.asarray(org)[None, :] + a[:, None] * u[None, :] + b[:, None] * v[None, :])
        nrms.append(np.broadcast_to(np.asarray(nrm), (a.size, 3)))
        face_id.append(np.full(a.size, f))
        obj_id.append(np.full(a.size, obj))
    perm = rng.permutation(sum(p.shape[0] for p in pts))
    return {"points": np.ascontiguousarray(np.concatenate(pts)[perm], np.float32),
            "normals": np.ascontiguousarray(np.concatenate(nrms)[perm], np.float32),
            "face": np.concatenate(face_id)[perm], "object": np.concatenate(obj_id)[perm], "spacing": h,
            "faces": len(faces), "objects": len(quads) + len(boxes)}


def segment_far_scene(seed=1, outliers=0):
    """A cloud whose neighbour sweeps take the far-query path of the grid (far_sweep.cuh): a dense blob (it sets a
    fine cell edge) inside sparse points spread over the unit cube, 2- and 3-fold duplicates, and optionally far
    outliers (kNN queries from them cross empty space). A radius of 0.3 spans ~19 cells of this grid. Normals: unit,
    scattered around +z. Returns (points, normals) float32, in random order."""
    rng = np.random.default_rng(seed)
    blob = 0.45 + 0.1 * rng.random((2000, 3))
    sparse = rng.random((400, 3))
    far = 0.5 + 30.0 * rng.standard_normal((outliers, 3))
    pts = np.concatenate([blob, sparse, far])
    pts = np.concatenate([pts, pts[:150], pts[2000:2060], pts[:40], pts[2400:2400 + outliers // 2]])
    nrm = np.array([0.0, 0.0, 1.0]) + 0.4 * rng.standard_normal(pts.shape)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    perm = rng.permutation(pts.shape[0])
    return pts[perm].astype(np.float32), nrm[perm].astype(np.float32)


def mean_shift_scene(blobs, per_blob, sigma=1.0, seed=1):
    """Truncated-Gaussian blobs for mean-shift: per_blob points around each centre, N(0, sigma^2) per axis, cut at
    4 sigma from the centre, point-symmetric about it (every offset d comes with -d), so the centre is the blob's
    centroid. Centres sit on a lattice of pitch 16 sigma around the origin with +-2 sigma jitter, hence >= 12 sigma
    apart. With the reference example's recipe (kernel radius 2 sigma, cluster tol 0.2 sigma) the answer is one
    cluster per blob. Returns dict(points (n,3) float32 in random order, blob (n,) blob id per point, centres
    (blobs,3) float64, sigma)."""
    rng = np.random.default_rng(seed)
    side = int(np.ceil(blobs ** (1.0 / 3.0)))
    lat = np.stack(np.meshgrid(*(np.arange(side),) * 3, indexing="ij"), axis=-1).reshape(-1, 3)[:blobs]
    centres = (lat - (side - 1) / 2.0) * 16.0 * sigma + rng.uniform(-2.0, 2.0, (blobs, 3)) * sigma
    half = (per_blob + 1) // 2
    off = rng.standard_normal((blobs, 4 * half, 3))
    keep = np.linalg.norm(off, axis=2) <= 4.0
    d = np.stack([o[k][:half] for o, k in zip(off, keep)]) * sigma  # (>= half of 4 * half survive the cut)
    pts = np.concatenate([centres[:, None, :] + d, centres[:, None, :] - d], axis=1)[:, :per_blob]
    blob = np.repeat(np.arange(blobs), per_blob)
    perm = rng.permutation(blobs * per_blob)
    return {"points": np.ascontiguousarray(pts.reshape(-1, 3)[perm], np.float32), "blob": blob[perm],
            "centres": centres, "sigma": float(sigma)}


def plane_scene(n, seed=1, noise=0.002, extent=4.0):
    """A room corner for plane RANSAC: a floor (~45 % of the points) and a wall (~25 %), each a square of side
    `extent` with truncated-Gaussian noise (sigma = noise, cut at 2.5 sigma) along its normal, plus ~30 % clutter
    uniform in the room's box. The scene is rotated by a random rigid transform. Returns dict(points (n,3) float32,
    labels (n,) 0 floor / 1 wall / 2 clutter, planes (2,4) float64 true (n0, n1, n2, d) of floor and wall,
    noise)."""
    rng = np.random.default_rng(seed)
    n_floor, n_wall = int(0.45 * n), int(0.25 * n)
    n_clut = n - n_floor - n_wall

    def slab(m):
        z = rng.standard_normal(4 * m + 8)
        return (z[np.abs(z) <= 2.5][:m]) * noise

    floor = np.column_stack([rng.uniform(0, extent, n_floor), rng.uniform(0, extent, n_floor), slab(n_floor)])
    wall = np.column_stack([rng.uniform(0, extent, n_wall), 0.5 * extent + slab(n_wall),
                            rng.uniform(0.05 * extent, 0.75 * extent, n_wall)])
    clutter = rng.uniform([0.0, 0.0, 0.05 * extent], [extent, extent, 0.75 * extent], (n_clut, 3))
    pts = np.concatenate([floor, wall, clutter])
    labels = np.concatenate([np.zeros(n_floor, np.int64), np.ones(n_wall, np.int64), np.full(n_clut, 2, np.int64)])
    T = np.asarray(rigid_from_axis_angle(rng.standard_normal(3), rng.uniform(0.2, 1.0), rng.uniform(-2, 2, 3)),
                   np.float64)
    R, t = T[:, :3], T[:, 3]
    pts = pts @ R.T + t
    planes = []
    for nrm, off in (((0.0, 0.0, 1.0), 0.0), ((0.0, 1.0, 0.0), -0.5 * extent)):
        nn = R @ np.array(nrm)
        planes.append(np.append(nn, off - nn @ t))
    perm = rng.permutation(n)
    return {"points": np.ascontiguousarray(pts[perm], np.float32), "labels": labels[perm], "planes": np.array(planes),
            "noise": float(noise)}


def warp_pair(n, seed=1, spacing=0.005, bend=0.01, noise=0.0005):
    """A non-rigid registration pair. dst: n points uniform on a smooth height field z = h(x, y) over a square of side
    L = spacing sqrt(n) (mean spacing `spacing`), with its analytic unit normals. src: every dst point moved by a
    smooth bend of amplitude `bend` (one period across the square in each coordinate), then by a small rigid offset
    (1 degree about a tilted axis, translation of 0.3 `bend` per axis), plus N(0, noise^2) noise per axis, in the same
    order as dst. Returns dict(dst, dst_normals, src (n,3) float32, spacing, side L)."""
    rng = np.random.default_rng(seed)
    L = spacing * np.sqrt(n)
    k = 2.0 * np.pi / L
    xy = rng.uniform(0.0, L, (n, 2))
    x, y = xy[:, 0], xy[:, 1]
    amp = 0.08 * L
    z = amp * np.sin(0.5 * k * x) * np.cos(0.5 * k * y)
    hx = amp * 0.5 * k * np.cos(0.5 * k * x) * np.cos(0.5 * k * y)
    hy = -amp * 0.5 * k * np.sin(0.5 * k * x) * np.sin(0.5 * k * y)
    dst = np.stack([x, y, z], 1)
    nrm = np.stack([-hx, -hy, np.ones(n)], 1)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    disp = bend * np.stack([np.sin(k * x), np.cos(k * y), np.sin(k * (x + y))], 1)
    ax = np.array([0.3, -0.2, 1.0]) / np.linalg.norm([0.3, -0.2, 1.0])
    th = np.deg2rad(1.0)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    R = np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K
    c = dst.mean(0)
    src = (dst + disp - c) @ R.T + c + 0.3 * bend * np.array([1.0, -1.0, 0.5]) + rng.normal(0.0, noise, (n, 3))
    return {"dst": np.ascontiguousarray(dst, np.float32), "dst_normals": np.ascontiguousarray(nrm, np.float32),
            "src": np.ascontiguousarray(src, np.float32), "spacing": float(spacing), "side": float(L)}


def sheet_color(x, y):
    """A smooth RGB texture over the plane (period ~0.2-0.35 along each axis), values in [0, 1]."""
    tau = 2 * np.pi
    return np.stack([0.5 + 0.5 * np.sin(tau * 4 * x) * np.cos(tau * 3 * y),
                     0.5 + 0.5 * np.cos(tau * 5 * x + 1.0) * np.sin(tau * 3 * y + 0.5),
                     0.5 + 0.5 * np.sin(tau * 3 * (x + y))], axis=1)


def textured_sheet_pair(n, seed=1, offset=(0.03, -0.02), relief=0.002):
    """Coloured-ICP stand-in: a low-relief sheet z = relief sin(7x) cos(6y) over [0,1)^2 with the colour texture
    sheet_color, sampled twice (independent uniform samples). The source is the second sample shifted in-plane by
    -offset, so the transform that registers it is a pure in-plane translation by +offset, which the geometry alone
    barely constrains and the colours do. Returns dict(dst, dst_normals, dst_colors, src, src_normals, src_colors, T_ref)."""
    rng = np.random.default_rng(seed)

    def sample():
        xy = rng.random((n, 2))
        x, y = xy[:, 0], xy[:, 1]
        z = relief * np.sin(7 * x) * np.cos(6 * y)
        g = np.stack([-7 * relief * np.cos(7 * x) * np.cos(6 * y), 6 * relief * np.sin(7 * x) * np.sin(6 * y),
                      np.ones(n)], axis=1)
        g /= np.linalg.norm(g, axis=1, keepdims=True)
        return np.stack([x, y, z], axis=1), g, sheet_color(x, y)

    dp, dn, dc = sample()
    sp, sn, sc = sample()
    sp = sp - np.array([offset[0], offset[1], 0.0])
    T_ref = np.hstack([np.eye(3), np.array([[offset[0]], [offset[1]], [0.0]])]).astype(np.float32)
    f = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731
    return dict(dst=f(dp), dst_normals=f(dn), dst_colors=f(dc), src=f(sp), src_normals=f(sn), src_colors=f(sc),
                T_ref=T_ref)
