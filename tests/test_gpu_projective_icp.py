"""Projective correspondence search of rigid ICP on the device (cb_icp_set_projection, DESIGN §4.21) against the numpy
fp32 restatement tests/projective_ref.py: correspondence lists bit for bit, sums within the fp bound of float64, the
device-resident loop against the host-driven loop and a float64 loop, detaching, residuals, argument errors and an
end-to-end tracking run over rendered frames."""
import numpy as np
import pytest

import depth_images_ref as dimg
import icp_ref
import projective_ref as pref
from cilantro_b200 import capi

pytestmark = pytest.mark.gpu

F = np.float32


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def k_for(w, h):
    f = F(0.8 * max(w, h))
    return np.array([[f, 0, (w - 1) / 2], [0, f, (h - 1) / 2], [0, 0, 1]], F)


def small_pose(seed, angle=0.02, shift=0.01):
    return dimg.pose(seed, angle, shift)


def inverse(T):
    T = np.asarray(T, np.float64)
    R = T[:, :3].T
    return np.hstack([R, (-R @ T[:, 3])[:, None]]).astype(F)


def scene(w, h, K, E=None, seed=0, special=True):
    """(dst, src, T): dst = a holed surface frame seen by the camera at pose E, with exact duplicates (z ties),
    non-finite points and points behind the camera; src = dst moved by the inverse of T plus noise, with points behind
    the camera, off the image and non-finite ones."""
    rng = np.random.default_rng(seed)
    depth = dimg.frame("holed", w, h, np.float32, seed=seed)
    dst, _, _ = dimg.depth_to_points(depth, K, 1000.0, None, None, E)
    dst = dst.reshape(-1, 3)
    if special and dst.shape[0]:
        dup = dst[rng.integers(0, dst.shape[0], max(1, dst.shape[0] // 10))]
        behind = dimg._rigid(E, np.array([[0.1, 0.2, -1.0]], F)) if E is not None else np.array([[0.1, 0.2, -1.0]], F)
        dst = np.vstack([dst, dup, [[np.nan, 0, 1], [np.inf, 0, 1], [0, 0, np.inf]], behind]).astype(F)
    T = small_pose(seed + 1)
    src = icp_ref.apply_f32(inverse(T), dst)
    src = (src + rng.normal(scale=0.002, size=src.shape)).astype(F)
    if special:
        extra = np.array([[0, 0, -2.0], [50.0, 0, 1.0], [np.nan, 1, 1], [1, np.inf, 1], [0, 0, 0]], F)
        src = np.vstack([src, extra]).astype(F)
    return dst, src, T


def clouds(ctx, dst, src, dst_n=None, src_n=None):
    return capi.Cloud(ctx, dst, dst_n), capi.Cloud(ctx, src, src_n)


def check_list(icp, dst, src, T, K, w, h, E, max_d2, fraction=1.0):
    icp.accumulate(T, metric="p2p", max_d2=max_d2, inlier_fraction=fraction)
    f, s, v = icp.correspondences()
    wf, ws, wv = pref.correspondences(dst, src, T, K, w, h, E, max_d2, fraction)
    assert np.array_equal(f, wf) and np.array_equal(s, ws), (f.size, wf.size)
    assert np.array_equal(v.view(np.uint32), wv.view(np.uint32))
    return f.size


@pytest.mark.parametrize("wh", [(1, 1), (31, 7), (33, 9), (640, 480), (1920, 1080)])
@pytest.mark.parametrize("general", [False, True])
def test_lists_match_restatement(ctx, wh, general):
    w, h = wh
    K = dimg.K_GENERAL if general else k_for(w, h)
    E = dimg.pose(7, 0.2, 0.1) if general else None
    dst, src, T = scene(w, h, K, E, seed=w + h)
    d, s = clouds(ctx, dst, src)
    icp = capi.Icp(ctx, d, s)
    icp.set_projection(K, w, h, E)
    total = 0
    for max_d2 in (F(1e-4), F(0.01), F(np.inf)):
        for TT in (T, icp_ref.identity().astype(F)):
            total += check_list(icp, dst, src, TT, K, w, h, E, max_d2)
    if w * h >= 640 * 480:
        assert total > 0
    for fraction in (0.5, 0.9):
        check_list(icp, dst, src, T, K, w, h, E, F(0.01), fraction)


def test_half_pixel_boundaries_and_ties(ctx):
    """K = I, z = 1: a point at x lands on llround(x). Exact halves round away from zero, (-0.5, 0) lands on pixel 0,
    -0.5 and w - 0.5 fall off; two destination points per pixel with the same z (the lower index wins) and a nearer
    one; values exactly at max_d2 are rejected."""
    w, h = 33, 9
    K = np.eye(3, dtype=F)
    gy, gx = np.mgrid[0:h, 0:w]
    grid = np.stack([gx.ravel(), gy.ravel(), np.ones(w * h)], 1).astype(F)
    nearer = grid[::5].copy()
    nearer[:, 2] = F(0.5)  # nearer points on the pixels (2x, 2y)
    dst = np.vstack([grid, grid[::3], nearer]).astype(F)  # grid[::3] ties exactly with lower-index originals
    xs = np.array([-0.75, -0.5, -0.49999997, -0.25, 0.5, 1.5, 2.5, 31.5, 32.4999, 32.5, 3.25, 7.75], F)
    src = np.stack([np.repeat(xs, h), np.tile(np.arange(h, dtype=F) + F(0.5), xs.size), np.ones(xs.size * h, F)], 1)
    src = np.vstack([src, grid[::7]]).astype(F)
    d, s = clouds(ctx, dst, src)
    icp = capi.Icp(ctx, d, s)
    icp.set_projection(K, w, h)
    T = icp_ref.identity().astype(F)
    for max_d2 in (F(0.25), F(0.5), F(0.5000001), F(1.0), F(np.inf)):
        check_list(icp, dst, src, T, K, w, h, None, max_d2)
    check_list(icp, dst, src, T, K, w, h, None, F(1.0), 0.3)


def test_empty_image_gives_no_correspondences(ctx):
    K = k_for(64, 48)
    dst, src, T = scene(64, 48, K, seed=3)
    d, s = clouds(ctx, dst, src)
    icp = capi.Icp(ctx, d, s)
    for w, h in ((0, 48), (64, 0), (0, 0)):
        icp.set_projection(K, w, h)
        sums = icp.accumulate(T, metric="p2p", max_d2=F(1.0))
        assert sums[0] == 0
        assert icp.correspondences()[0].size == 0
        r = icp.estimate(metric="p2p", max_iter=3, tol=0.0, max_d2=F(1.0), T_init=T)
        assert r["num_corr"] == 0


def combined_sums(dst, dst_n, src, src_n, T, first, second, w_pt, w_pl, wc_pt=None, wc_pl=None, values=None):
    """The 28 values of the combined pass (n, upper AtA row-major, Atb) in float64 from the fp32 inputs."""
    Tf = np.asarray(T, F)
    dm = dst[icp_ref.finite_rows(dst)].astype(np.float64).mean(0).astype(F)
    sm = icp_ref.apply_f32(Tf, src[icp_ref.finite_rows(src)].astype(np.float64).mean(0).astype(F)[None])[0]
    d = (dst[first] - dm).astype(np.float64)
    q = icp_ref.apply_f32(Tf, src[second])
    s = (q - sm).astype(np.float64)
    v, e = d + s, d - s
    A, b = np.zeros((6, 6)), np.zeros(6)
    wp = np.full(len(first), w_pt) if wc_pt is None else (F(w_pt) * np.exp(F(wc_pt) * values)).astype(np.float64)
    wl = np.full(len(first), w_pl) if wc_pl is None else (F(w_pl) * np.exp(F(wc_pl) * values)).astype(np.float64)
    if w_pt > 0:
        for k in range(len(first)):
            vx = np.array([[0, -v[k, 2], v[k, 1]], [v[k, 2], 0, -v[k, 0]], [-v[k, 1], v[k, 0], 0]])
            E = np.vstack([vx, np.eye(3)])  # eq_vecs: E E^T and E e as the pass forms them
            A += wp[k] * E @ E.T
            b += wp[k] * E @ e[k]
    if w_pl > 0:
        n = dst_n[first].astype(np.float64)
        if src_n is not None:
            n = n + src_n[second].astype(np.float64) @ Tf[:, :3].astype(np.float64).T
        a = np.hstack([np.cross(v, n), n])
        r = (n * e).sum(1)
        A += (wl[:, None] * a).T @ a
        b += (wl[:, None] * a).T @ r
    iu = np.triu_indices(6)
    return np.concatenate([[len(first)], A[iu], b])


@pytest.mark.parametrize("case", ["p2p", "combined", "symmetric", "rbf"])
def test_sums_within_fp_bound(ctx, case):
    w, h = 160, 120
    K = k_for(w, h)
    depth = dimg.frame("full", w, h, np.float32, seed=4)
    dst, dst_n, _ = dimg.depth_to_points(depth, K, 1000.0, None, None, None, normals=True)
    T = small_pose(5)
    src = icp_ref.apply_f32(inverse(T), dst)
    src_n = (dst_n @ np.asarray(T, np.float64)[:, :3]).astype(F)
    d, s = clouds(ctx, dst, src, dst_n, src_n if case == "symmetric" else None)
    icp = capi.Icp(ctx, d, s)
    icp.set_projection(K, w, h)
    max_d2 = F(1e-3)
    first, second, values = pref.correspondences(dst, src, T, K, w, h, None, max_d2)
    assert first.size > 1000
    if case == "p2p":
        got = icp.accumulate(T, metric="p2p", max_d2=max_d2)
        dd = dst[first].astype(np.float64)
        q = icp_ref.apply_f32(T, src[second]).astype(np.float64)
        want = np.concatenate([[first.size], dd.sum(0), q.sum(0), (dd[:, :, None] * q[:, None, :]).sum(0).ravel()])
    else:
        kw = dict(w_pt=0.1, w_pl=1.0)
        if case == "rbf":
            kw.update(pt_rbf_sigma=0.02, pl_rbf_sigma=0.02)
        got = icp.accumulate(T, metric="combined", max_d2=max_d2, **kw)
        coeff = capi.rbf_coeff(0.02) if case == "rbf" else None
        want = combined_sums(dst, dst_n, src, src_n if case == "symmetric" else None, T, first, second, 0.1, 1.0,
                             coeff, coeff, values)
    assert got[0] == want[0]
    scale = np.abs(want).max()
    assert np.abs(got - want).max() <= 1e-5 * scale, np.abs(got - want).max() / scale


def loop_scene(ctx, w=320, h=240, seed=6, symmetric=False):
    K = k_for(w, h)
    depth = dimg.frame("full", w, h, np.float32, seed=seed)
    dst, dst_n, _ = dimg.depth_to_points(depth, K, 1000.0, None, None, None, normals=True)
    T = small_pose(seed + 1, 0.03, 0.02)
    src = icp_ref.apply_f32(inverse(T), dst)
    src_n = (dst_n @ np.asarray(T, np.float64)[:, :3]).astype(F)
    d, s = clouds(ctx, dst, src, dst_n, src_n if symmetric else None)
    return K, dst, dst_n, src, src_n, T, d, s


@pytest.mark.parametrize("metric", ["p2p", "combined", "symmetric"])
def test_device_loop_matches_host_loop_and_float64(ctx, metric):
    K, dst, dst_n, src, src_n, T, d, s = loop_scene(ctx, symmetric=metric == "symmetric")
    w, h = 320, 240
    icp = capi.Icp(ctx, d, s)
    icp.set_projection(K, w, h)
    kw = dict(metric="p2p") if metric == "p2p" else dict(metric="combined", w_pt=0.1, w_pl=1.0)
    max_d2 = F(0.02 ** 2)
    dev = icp.estimate(max_iter=5, tol=0.0, max_d2=max_d2, timing=0, **kw)
    again = icp.estimate(max_iter=5, tol=0.0, max_d2=max_d2, timing=0, **kw)
    assert np.array_equal(dev["T"], again["T"])
    assert again["kernel_launches"] == 2 * again["iterations"] == 10  # projective pass + finish kernel
    host = icp.estimate(max_iter=5, tol=0.0, max_d2=max_d2, host_loop=True, **kw)
    assert host["iterations"] == dev["iterations"] and host["num_corr"] == dev["num_corr"]
    assert np.abs(host["T"] - dev["T"]).max() < 1e-5
    want = pref.icp_loop(dst, src, K, w, h, None, icp_ref.identity(), 5, max_d2,
                         metric="p2p" if metric == "p2p" else "combined", dst_n=dst_n,
                         src_n=src_n if metric == "symmetric" else None, w_pt=0.1, w_pl=1.0)
    assert np.abs(dev["T"] - want).max() < 1e-5
    # cb_icp_correspondences re-runs the per-query search (projective_search_kernel) at the transform the last
    # iteration used: its size is the device pass's count, and its list is the restatement's
    f, s2, _ = icp.correspondences()
    assert f.size == dev["num_corr"]
    with pytest.raises(capi.CbError):
        icp.loop_cache()


@pytest.mark.parametrize("metric", ["p2p", "combined"])
def test_device_pass_accumulates_the_restated_list(ctx, metric):
    """One device-loop iteration from several starting transforms: icp_projective_kernel's correspondence count equals
    the restated list's size, and its step equals the host loop's, whose passes accumulate the per-query result that
    the list tests pin bit for bit."""
    K, dst, dst_n, src, src_n, T, d, s = loop_scene(ctx, 320, 240, seed=13)
    icp = capi.Icp(ctx, d, s)
    icp.set_projection(K, 320, 240)
    kw = dict(metric="p2p") if metric == "p2p" else dict(metric="combined", w_pt=0.1, w_pl=1.0)
    max_d2 = F(0.02 ** 2)
    for k, T0 in enumerate((icp_ref.identity().astype(F), T, small_pose(40, 0.01, 0.005), small_pose(41, 0.03, 0.01))):
        dev = icp.estimate(max_iter=1, tol=0.0, max_d2=max_d2, T_init=T0, **kw)
        host = icp.estimate(max_iter=1, tol=0.0, max_d2=max_d2, T_init=T0, host_loop=True, **kw)
        f, _, _ = pref.correspondences(dst, src, T0, K, 320, 240, None, max_d2)
        assert dev["num_corr"] == host["num_corr"] == f.size, (k, dev["num_corr"], f.size)
        assert np.abs(dev["T"] - host["T"]).max() < 1e-6, k


def test_device_loop_iteration_edges_and_convergence(ctx):
    K, dst, dst_n, src, src_n, T, d, s = loop_scene(ctx, 160, 120, seed=8)
    icp = capi.Icp(ctx, d, s)
    icp.set_projection(K, 160, 120)
    max_d2 = F(0.02 ** 2)
    T0 = icp_ref.identity().astype(F)
    r0 = icp.estimate(metric="p2p", max_iter=0, max_d2=max_d2)
    assert r0["iterations"] == 0 and np.array_equal(r0["T"], T0)
    r1 = icp.estimate(metric="p2p", max_iter=1, tol=0.0, max_d2=max_d2)
    h1 = icp.estimate(metric="p2p", max_iter=1, tol=0.0, max_d2=max_d2, host_loop=True)
    assert r1["iterations"] == 1 and np.abs(r1["T"] - h1["T"]).max() < 1e-6
    # the convergence rule: stop at the first update whose norm is below tol, on both loops
    for tol in (1.0, 1e-4):
        a = icp.estimate(metric="combined", max_iter=30, tol=tol, max_d2=max_d2, w_pt=0.1)
        b = icp.estimate(metric="combined", max_iter=30, tol=tol, max_d2=max_d2, w_pt=0.1, host_loop=True)
        assert a["converged"] and a["iterations"] == b["iterations"]
        assert a["last_delta"] < tol
    assert icp.estimate(metric="combined", max_iter=30, tol=1.0, max_d2=max_d2, w_pt=0.1)["iterations"] == 1


def test_inner_gauss_newton_steps_and_fraction_take_the_host_paths(ctx):
    K, dst, dst_n, src, src_n, T, d, s = loop_scene(ctx, 160, 120, seed=9)
    icp = capi.Icp(ctx, d, s)
    icp.set_projection(K, 160, 120)
    max_d2 = F(0.02 ** 2)
    r = icp.estimate(metric="combined", max_iter=3, tol=0.0, max_d2=max_d2, max_opt_iter=3, opt_tol=0.0)
    assert r["iterations"] == 3 and np.isfinite(r["T"]).all()
    icp.estimate(metric="p2p", max_iter=1, tol=0.0, max_d2=max_d2, inlier_fraction=0.7)
    f, s2, v = icp.correspondences()
    wf, ws, wv = pref.correspondences(dst, src, icp_ref.identity().astype(F), K, 160, 120, None, max_d2, 0.7)
    assert np.array_equal(f, wf) and np.array_equal(s2, ws) and np.array_equal(v.view(np.uint32), wv.view(np.uint32))


def test_detach_restores_kdtree_and_residuals_stay_kdtree(ctx):
    K, dst, dst_n, src, src_n, T, d, s = loop_scene(ctx, 160, 120, seed=10)
    kw = dict(metric="combined", w_pt=0.1, max_iter=4, tol=0.0, max_d2=F(0.02 ** 2))
    plain = capi.Icp(ctx, d, s)
    want = plain.estimate(**kw)
    want_host = plain.estimate(host_loop=True, **kw)
    want_res = plain.residuals(T, metric="combined", w_pt=0.1)
    icp = capi.Icp(ctx, d, s)
    icp.set_projection(K, 160, 120)
    proj = icp.estimate(**kw)
    assert np.array_equal(icp.residuals(T, metric="combined", w_pt=0.1).view(np.uint32), want_res.view(np.uint32))
    icp.set_projection(None, 0, 0)
    got = icp.estimate(**kw)
    assert np.array_equal(got["T"], want["T"]) and got["num_corr"] == want["num_corr"]
    icp.loop_cache()  # the kd-tree device loop ran again
    assert np.array_equal(icp.estimate(host_loop=True, **kw)["T"], want_host["T"])
    assert not np.array_equal(proj["T"], got["T"])


def test_argument_errors(ctx):
    K, dst, dst_n, src, src_n, T, d, s = loop_scene(ctx, 64, 48, seed=11)
    icp = capi.Icp(ctx, d, s)
    bad = K.copy()
    bad[0, 0] = np.nan
    with pytest.raises(capi.CbError):
        icp.set_projection(bad, 64, 48)
    with pytest.raises(capi.CbError):
        icp.set_projection(K, 64, 48, np.full((3, 4), np.inf, F))
    with pytest.raises(capi.CbError):
        icp.set_projection(K, 1 << 16, 1 << 16)
    icp.set_projection(K, 64, 48)
    for kw in (dict(search_dir="both"), dict(search_dir="first_to_second"), dict(require_reciprocal=True),
               dict(one_to_one=True)):
        with pytest.raises(capi.CbError):
            icp.estimate(metric="p2p", max_iter=2, **kw)
        with pytest.raises(capi.CbError):
            icp.accumulate(T, metric="p2p", **kw)
    icp.set_features("point_normal", dst_normals=dst_n, src_normals=src_n)
    with pytest.raises(capi.CbError):
        icp.estimate(metric="p2p", max_iter=2)
    icp.set_features("point")
    icp.estimate(metric="p2p", max_iter=2)


def test_no_device_memory_growth(ctx):
    import torch

    K, dst, dst_n, src, src_n, T, d, s = loop_scene(ctx, 320, 240, seed=12)
    icp = capi.Icp(ctx, d, s)
    for k in range(3):
        icp.set_projection(K, 320, 240)
        icp.estimate(metric="combined", max_iter=4, max_d2=F(4e-4))
    ctx.synchronize()
    free0 = torch.cuda.mem_get_info(0)[0]
    for k in range(20):
        icp.set_projection(K, 320, 240)
        icp.estimate(metric="combined", max_iter=4, max_d2=F(4e-4))
        icp.estimate(metric="combined", max_iter=2, max_d2=F(4e-4), host_loop=True)
        icp.accumulate(T, metric="p2p", max_d2=F(4e-4), inlier_fraction=0.5)
    ctx.synchronize()
    assert free0 - torch.cuda.mem_get_info(0)[0] <= 8 << 20


def room(spacing=0.01):
    """Points of a 4 x 2.4 x 5 m room (floor, ceiling, three walls) and two boxes, with their normals."""
    pts, nrm = [], []

    def plane(o, u, v, nu, nv, n):
        a, b = np.meshgrid(np.arange(nu) * spacing, np.arange(nv) * spacing)
        p = np.asarray(o) + a.reshape(-1, 1) * np.asarray(u) + b.reshape(-1, 1) * np.asarray(v)
        pts.append(p)
        nrm.append(np.tile(n, (p.shape[0], 1)))

    X, Y, Z = 4.0, 2.4, 5.0
    nx, ny, nz = int(X / spacing), int(Y / spacing), int(Z / spacing)
    plane([-2, 1.2, 0], [1, 0, 0], [0, 0, 1], nx, nz, [0, -1, 0])    # floor
    plane([-2, -1.2, 0], [1, 0, 0], [0, 0, 1], nx, nz, [0, 1, 0])    # ceiling
    plane([-2, -1.2, 5], [1, 0, 0], [0, 1, 0], nx, ny, [0, 0, -1])   # back wall
    plane([-2, -1.2, 0], [0, 1, 0], [0, 0, 1], ny, nz, [1, 0, 0])    # left wall
    plane([2, -1.2, 0], [0, 1, 0], [0, 0, 1], ny, nz, [-1, 0, 0])    # right wall
    for cx, cz, sz in ((-0.8, 3.0, 0.6), (0.9, 3.6, 0.8)):
        plane([cx, 1.2 - sz, cz - sz / 2], [1, 0, 0], [0, 1, 0], int(sz / spacing), int(sz / spacing), [0, 0, -1])
        plane([cx, 1.2 - sz, cz - sz / 2], [0, 0, 1], [0, 1, 0], int(sz / spacing), int(sz / spacing), [-1, 0, 0])
        plane([cx, 1.2 - sz, cz - sz / 2], [1, 0, 0], [0, 0, 1], int(sz / spacing), int(sz / spacing), [0, -1, 0])
    return np.vstack(pts).astype(F), np.vstack(nrm).astype(F)


def test_tracking_rendered_frames(ctx):
    """The fusion localisation loop: frames rendered from a trajectory, converted back with normals on the device and
    tracked against the first frame's cloud with the reference example's settings."""
    w, h = 640, 480
    K = np.array([[528, 0, 320], [0, 528, 240], [0, 0, 1]], F)
    world, _ = room()
    conv = capi.DepthConverter(np.float32, 1.0)
    poses = [dimg.pose(100 + k, 0.004 * k, 0.0) for k in range(6)]
    for k, P in enumerate(poses):
        P[:, 3] = [0.01 * k, -0.005 * k, 0.02 * k]
    frames = []
    for P in poses:
        depth = capi.points_to_depth_image(ctx, world, K, w, h, conv, extrinsics=P)
        frames.append(capi.depth_image_to_points(ctx, depth, K, conv, normals=True, to_device=True)["cloud"])
    model_host = capi.depth_image_to_points(ctx, capi.points_to_depth_image(ctx, world, K, w, h, conv, extrinsics=poses[0]),
                                            K, conv, normals=True, extrinsics=poses[0])
    model = capi.Cloud(ctx, model_host["points"], model_host["normals"])
    pose = poses[0].copy()
    worst = 0.0
    for k in range(1, len(poses)):
        icp = capi.Icp(ctx, model, frames[k])
        icp.set_projection(K, w, h, pose)
        r = icp.estimate(metric="combined", w_pt=0.0, w_pl=1.0, max_d2=F(0.1 * 0.1), T_init=pose, tol=5e-4, max_iter=6)
        pose = r["T"]
        err = float(np.abs(pose.astype(np.float64) - poses[k]).max())
        worst = max(worst, err)
        print(f"frame {k}: {r['iterations']} iterations, {r['num_corr']} correspondences, pose error {err:.2e}")
    assert worst < 1e-3, worst
