"""numpy fp32 restatement of the depth-image <-> cloud conversions (DESIGN §4.20): every product, sum and quotient is
one float32 operation in the order written there, so the device results must equal these bit for bit.

Images are [h, w] (rgb [h, w, 3] uint8), pixel k = y * w + x; intrinsics K are 3 x 3, extrinsics [R | t] 3 x 4."""
import numpy as np

F = np.float32


def dot(a0, a1, a2, b0, b1, b2):
    """Eigen's dot of two 3-vectors: (a0 b0 + a1 b1) + a2 b2."""
    return (F(a0) * F(b0) + F(a1) * F(b1)) + F(a2) * F(b2)


def inverse3(K):
    """intrinsics.inverse() as Eigen 3.4 forms it for a fixed 3 x 3: cofactors, det from the first column, one
    reciprocal, then inverse(i, j) = C(j, i) * invdet."""
    m = np.asarray(K, F).reshape(3, 3)

    def cof(i, j):
        i1, i2, j1, j2 = (i + 1) % 3, (i + 2) % 3, (j + 1) % 3, (j + 2) % 3
        return m[i1, j1] * m[i2, j2] - m[i1, j2] * m[i2, j1]

    with np.errstate(all="ignore"):
        det = dot(cof(0, 0), cof(1, 0), cof(2, 0), m[0, 0], m[1, 0], m[2, 0])
        invdet = F(1.0) / det
        return np.array([[cof(j, i) * invdet for j in range(3)] for i in range(3)], F)


def _rows(A, v0, v1, v2):
    return np.stack([dot(A[i, 0], A[i, 1], A[i, 2], v0, v1, v2) for i in range(3)], -1)


def _rigid(T, p, translate=True):
    T = np.asarray(T, F).reshape(3, 4)
    q = _rows(T[:, :3], p[..., 0], p[..., 1], p[..., 2])
    return q + T[:, 3] if translate else q


def metric_depth(raw, scale=1.0, max_depth=None):
    """getMetricValue of DepthValueConverter / TruncatedDepthValueConverter: inverseScale * float(raw), then 0 at or
    above max_depth."""
    inv = F(1.0) / F(scale)
    z = inv * np.asarray(raw).astype(F)
    if max_depth is not None:
        z = np.where(z < F(max_depth), z, F(0.0)).astype(F)
    return z


def normals_of(p):
    """Per-pixel normal of a [h, w, 3] back-projected grid: (p[y+1] - p[y-1]) x (p[x+1] - p[x-1]), normalised as
    Eigen's normalized(), for interior pixels whose four neighbours and itself have z > 0; NaN elsewhere."""
    h, w, _ = p.shape
    n = np.full_like(p, np.nan)
    if h < 3 or w < 3:
        return n
    c, up, dn, lf, rt = p[1:-1, 1:-1], p[:-2, 1:-1], p[2:, 1:-1], p[1:-1, :-2], p[1:-1, 2:]
    ok = (c[..., 2] > 0) & (rt[..., 2] > 0) & (lf[..., 2] > 0) & (dn[..., 2] > 0) & (up[..., 2] > 0)
    a, b = dn - up, rt - lf
    cr = np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                   a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)
    s = (cr[..., 0] * cr[..., 0] + cr[..., 1] * cr[..., 1]) + cr[..., 2] * cr[..., 2]
    pos = s > 0
    r = np.sqrt(np.where(pos, s, F(1.0))).astype(F)
    cr = np.where(pos[..., None], cr / r[..., None], cr)
    n[1:-1, 1:-1] = np.where(ok[..., None], cr, F(np.nan))
    return n


def depth_to_points(depth, K, scale=1.0, max_depth=None, rgb=None, extrinsics=None, normals=False, keep_invalid=False):
    """depthImageToPoints / ...Normals / RGBDImagesToPointsColors / ...NormalsColors, with or without extrinsics.
    Returns (points, normals or None, colors or None) as [m, 3] float32 arrays."""
    with np.errstate(all="ignore"):
        depth = np.asarray(depth)
        h, w = depth.shape
        z = metric_depth(depth, scale, max_depth)
        x = np.arange(w, dtype=np.float64).astype(F)[None, :]
        y = np.arange(h, dtype=np.float64).astype(F)[:, None]
        v0, v1 = z * x, z * y
        Ki = inverse3(K)
        A = Ki
        post = extrinsics is not None
        if post and keep_invalid and not normals:
            # (extrinsics * intrinsics_inv) * v: the isometry takes the 3 x 3 matrix's columns as points
            T = np.asarray(extrinsics, F).reshape(3, 4)
            A = np.array([[T[i, 3] + dot(T[i, 0], T[i, 1], T[i, 2], Ki[0, j], Ki[1, j], Ki[2, j]) for j in range(3)]
                          for i in range(3)], F)
            post = False
        p = _rows(A, v0, v1, z)
        n = normals_of(p) if normals else None
        keep = (~np.isnan(n[..., 0]) if normals else p[..., 2] > 0).reshape(-1)
        p = p.reshape(-1, 3)
        n = None if n is None else n.reshape(-1, 3)
        c = None
        if rgb is not None:
            c = F(1.0) / F(255.0) * np.asarray(rgb, np.uint8).reshape(-1, 3).astype(F)
        if not keep_invalid:
            p = p[keep]
            n = None if n is None else n[keep]
            c = None if c is None else c[keep]
        if post:
            p = _rigid(extrinsics, p)
            n = None if n is None else _rigid(extrinsics, n, translate=False)
        return p.astype(F), (None if n is None else n.astype(F)), (None if c is None else c.astype(F))


def _round_half_away(v):
    r = np.trunc(v)
    f = v - r
    return r + np.where(f >= 0.5, 1.0, 0.0) - np.where(f <= -0.5, 1.0, 0.0)


def _project(points, K, extrinsics, w, h):
    """(camera-frame z, pixel index or -1) of every point: extrinsics.inverse() applied as linear p + translation,
    z <= 0 and non-finite projections skipped, llround (half away from zero) and the image bounds."""
    with np.errstate(all="ignore"):
        p = np.asarray(points, F).reshape(-1, 3)
        if extrinsics is not None:
            T = np.asarray(extrinsics, F).reshape(3, 4)
            L = T[:, :3].T.copy()
            tr = -np.array([dot(L[i, 0], L[i, 1], L[i, 2], T[0, 3], T[1, 3], T[2, 3]) for i in range(3)], F)
            p = _rows(L, p[:, 0], p[:, 1], p[:, 2]) + tr
        K = np.asarray(K, F).reshape(3, 3)
        z = p[:, 2]
        inv_z = F(1.0) / z
        fx = inv_z * dot(K[0, 0], K[0, 1], K[0, 2], p[:, 0], p[:, 1], p[:, 2])
        fy = inv_z * dot(K[1, 0], K[1, 1], K[1, 2], p[:, 0], p[:, 1], p[:, 2])
        ok = (z > 0) & np.isfinite(fx) & np.isfinite(fy)
        rx = _round_half_away(np.where(ok, fx, 0).astype(np.float64))
        ry = _round_half_away(np.where(ok, fy, 0).astype(np.float64))
        ok &= (rx >= 0) & (ry >= 0) & (rx < w) & (ry < h)
        pix = np.where(ok, ry * w + rx, -1).astype(np.int64)
        return z, pix


def raw_depth(z, dtype, scale=1.0, max_depth=None):
    """getRawValue: (raw, writes) per point. An unsigned short that does not fit is skipped; raw 0 never writes."""
    with np.errstate(all="ignore"):
        v = F(scale) * np.asarray(z, F)
        ok = np.ones(v.shape, bool) if max_depth is None else (np.asarray(z, F) < F(max_depth))
        if np.dtype(dtype) == np.uint16:
            ok &= (v >= 0) & (v < 65536)
            raw = np.where(ok, np.trunc(np.where(ok, v, 0)), 0).astype(np.uint16)
        else:
            ok &= v > 0
            raw = np.where(ok, v, 0).astype(F)
        return raw, ok & (raw > 0)


def color_bytes(c):
    """static_cast<unsigned char>(255.0f * c), saturated: NaN and values <= 0 give 0, values >= 255 give 255."""
    with np.errstate(all="ignore"):
        v = F(255.0) * np.asarray(c, F)
        return np.where(v > 0, np.where(v >= 255, 255, np.trunc(np.where(v > 0, v, 0))), 0).astype(np.uint8)


def _winners(pix, key, npix):
    """Serial z-buffer: per pixel the smallest key, the lowest point index on ties; -1 where no point lands."""
    win = np.full(npix, -1, np.int64)
    idx = np.nonzero(pix >= 0)[0]
    if idx.size:
        order = np.lexsort((idx, key[idx], pix[idx]))
        sp = pix[idx][order]
        first = np.ones(sp.size, bool)
        first[1:] = sp[1:] != sp[:-1]
        win[sp[first]] = idx[order][first]
    return win


def points_to_depth_image(points, K, w, h, dtype=np.uint16, scale=1.0, max_depth=None, colors=None, extrinsics=None):
    """pointsToDepthImage / pointsColorsToRGBDImages: the [h, w] depth image (and [h, w, 3] rgb with colors)."""
    z, pix = _project(points, K, extrinsics, w, h)
    raw, ok = raw_depth(z, dtype, scale, max_depth)
    pix = np.where(ok, pix, -1)
    win = _winners(pix, raw.astype(np.float64), w * h)
    depth = np.zeros(w * h, dtype)
    hit = win >= 0
    depth[hit] = raw[win[hit]]
    if colors is None:
        return depth.reshape(h, w)
    rgb = np.zeros((w * h, 3), np.uint8)
    rgb[hit] = color_bytes(np.asarray(colors, F).reshape(-1, 3)[win[hit]])
    return depth.reshape(h, w), rgb.reshape(h, w, 3)


def points_to_index_map(points, K, w, h, extrinsics=None):
    """pointsToIndexMap: per pixel the index of the smallest camera-frame z (lowest index on ties), 2^64 - 1 where
    empty."""
    z, pix = _project(points, K, extrinsics, w, h)
    win = _winners(pix, z.astype(np.float64), w * h)
    out = np.full(w * h, np.iinfo(np.uint64).max, np.uint64)
    out[win >= 0] = win[win >= 0].astype(np.uint64)
    return out.reshape(h, w)


# ---- seeded inputs shared by the restatement and device tests -------------------------------------------------------
K_PINHOLE = np.array([[525.0, 0.0, 319.5], [0.0, 525.0, 239.5], [0.0, 0.0, 1.0]], F)
# skew and a last row other than (0, 0, 1)
K_GENERAL = np.array([[410.0, 3.5, 20.25], [0.0, 395.0, 11.75], [0.001, -0.002, 1.25]], F)


def pose(seed, angle=0.3, shift=0.2):
    """A seeded rigid transform [R | t] (3 x 4 float32)."""
    rng = np.random.default_rng(seed)
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    Kx = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    R = np.eye(3) + np.sin(angle) * Kx + (1 - np.cos(angle)) * Kx @ Kx
    return np.hstack([R, rng.normal(scale=shift, size=(3, 1))]).astype(F)


def frame(kind, w, h, dtype, seed=0):
    """A seeded raw depth image: 'zero', 'single' (one valid pixel), 'full' (all valid, a smooth surface), 'holed'
    (random holes), 'special' (float: NaN, +-Inf, negative values, and for both types the largest raw value)."""
    rng = np.random.default_rng(seed)
    dt = np.dtype(dtype)
    yy, xx = np.mgrid[0:h, 0:w]
    surf = 1.5 + 0.3 * np.sin(xx / 17.0) * np.cos(yy / 23.0) + 0.001 * (xx + yy)
    img = (surf * 1000.0).astype(np.uint16) if dt == np.uint16 else (surf * 1000.0).astype(F)
    if kind == "zero":
        img[:] = 0
    elif kind == "single":
        v = img[h // 2, w // 2]
        img[:] = 0
        img[h // 2, w // 2] = v
    elif kind == "holed":
        img[rng.random((h, w)) < 0.2] = 0
    elif kind == "special":
        r = rng.random((h, w))
        if dt == np.uint16:
            img[r < 0.1] = 65535
            img[(r >= 0.1) & (r < 0.2)] = 0
        else:
            img[r < 0.05] = np.nan
            img[(r >= 0.05) & (r < 0.1)] = np.inf
            img[(r >= 0.1) & (r < 0.15)] = -np.inf
            img[(r >= 0.15) & (r < 0.25)] *= -1
            img[(r >= 0.25) & (r < 0.3)] = np.finfo(F).max
    return img


def rgb_frame(w, h, seed=0):
    return np.random.default_rng(seed + 99).integers(0, 256, (h, w, 3), dtype=np.uint8)
