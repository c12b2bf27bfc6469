"""Depth-image and RGB-D <-> cloud conversions on the device (cb_depth_image_to_points, cb_points_to_depth_image,
cb_points_to_index_map) against the numpy fp32 restatement of DESIGN §4.20 (tests/depth_images_ref.py), bit for bit:
points, normals with their NaN pattern, colours, counts, depth and rgb images and index maps."""
import numpy as np
import pytest

import depth_images_ref as ref
from cilantro_b200 import capi

pytestmark = pytest.mark.gpu

DTYPES = [np.uint16, np.float32]
# (scale, max_depth): DepthValueConverter and TruncatedDepthValueConverter, the latter cutting through the frames
CONVERTERS = [(1000.0, None), (1000.0, 1.6)]
SMALL = [(1, 1), (9, 1), (1, 9), (2, 2), (3, 3), (31, 7), (32, 8), (33, 9), (65, 17)]
KINDS = ["zero", "single", "full", "holed", "special"]


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def bits(a):
    """The bits of a float32 array with every NaN in one encoding: the device writes NaNs with another payload than
    numpy's, so the NaN pattern is compared by position."""
    a = np.ascontiguousarray(a, np.float32)
    return np.where(np.isnan(a), np.float32(np.nan), a).view(np.uint32)


def check_back(ctx, depth, K, scale, max_depth, rgb, T, normals, keep):
    conv = capi.DepthConverter(depth.dtype, scale, max_depth)
    got = capi.depth_image_to_points(ctx, depth, K, conv, rgb=rgb, extrinsics=T, normals=normals, keep_invalid=keep)
    p, n, c = ref.depth_to_points(depth, K, scale, max_depth, rgb, T, normals, keep)
    assert got["count"] == p.shape[0]
    assert np.array_equal(bits(got["points"]), bits(p))
    if normals:
        assert np.array_equal(bits(got["normals"]), bits(n))
    if rgb is not None:
        assert np.array_equal(bits(got["colors"]), bits(c))
    return got


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("conv", CONVERTERS)
@pytest.mark.parametrize("normals", [False, True])
@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("extrinsics", [False, True])
def test_back_projection_small(ctx, dtype, conv, normals, keep, extrinsics):
    T = ref.pose(3) if extrinsics else None
    for w, h in SMALL:
        for kind in KINDS:
            depth = ref.frame(kind, w, h, dtype, seed=w + 7 * h)
            rgb = ref.rgb_frame(w, h, seed=w)
            for K in (ref.K_PINHOLE, ref.K_GENERAL):
                check_back(ctx, depth, K, *conv, None, T, normals, keep)
                check_back(ctx, depth, K, *conv, rgb, T, normals, keep)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("wh", [(640, 480), (1920, 1080)])
def test_back_projection_full_frames(ctx, dtype, wh):
    w, h = wh
    T = ref.pose(11)
    rgb = ref.rgb_frame(w, h, seed=2)
    for kind in ("holed", "special", "full"):
        depth = ref.frame(kind, w, h, dtype, seed=w)
        for normals in (False, True):
            for keep in (False, True):
                check_back(ctx, depth, ref.K_PINHOLE, 1000.0, None, rgb, T if keep else None, normals, keep)
    check_back(ctx, ref.frame("holed", w, h, dtype), ref.K_GENERAL, 1000.0, 1.6, None, T, True, False)


def test_depth_at_max_depth_and_largest_raw(ctx):
    # 1600 / 1000 = 1.6 exactly at the cut (truncated to 0), 65535 kept below a larger cut
    depth = np.full((5, 6), 1600, np.uint16)
    depth[2, 3] = 65535
    for md in (1.6, 70.0):
        check_back(ctx, depth, ref.K_PINHOLE, 1000.0, md, None, None, True, True)
        check_back(ctx, depth, ref.K_PINHOLE, 1000.0, md, None, None, False, False)
    f = np.full((4, 4), 1.6, np.float32)
    got = check_back(ctx, f, ref.K_PINHOLE, 1.0, 1.6, None, None, False, False)
    assert got["count"] == 0


def test_zero_cross_product_keeps_a_zero_normal(ctx):
    depth = np.full((4, 5), 1e-25, np.float32)
    got = check_back(ctx, depth, ref.K_PINHOLE, 1.0, None, None, None, True, False)
    assert got["count"] == 6 and np.all(got["normals"] == 0)


class CudaImage:
    """A torch CUDA tensor seen as an array of another dtype of the same size (torch has no CUDA uint16 copies)."""

    def __init__(self, t, dtype):
        self.t, self.shape = t, tuple(t.shape)
        self.__cuda_array_interface__ = dict(t.__cuda_array_interface__, typestr=np.dtype(dtype).str)


def test_device_input_equals_host_input(ctx):
    torch = pytest.importorskip("torch")
    w, h = 333, 201
    for dtype in DTYPES:
        depth = ref.frame("holed", w, h, dtype, seed=5)
        rgb = ref.rgb_frame(w, h)
        conv = capi.DepthConverter(dtype, 1000.0)
        held = torch.from_numpy(depth.view(np.int16) if dtype == np.uint16 else depth).cuda()
        dd = CudaImage(held, depth.dtype)
        dr = torch.from_numpy(rgb).cuda()
        a = capi.depth_image_to_points(ctx, depth, ref.K_PINHOLE, conv, rgb=rgb, normals=True)
        b = capi.depth_image_to_points(ctx, dd, ref.K_PINHOLE, conv, rgb=dr, normals=True)
        for key in ("points", "normals", "colors"):
            assert np.array_equal(bits(a[key]), bits(b[key]))


def test_cloud_output_equals_host_output(ctx):
    w, h = 160, 120
    depth = ref.frame("holed", w, h, np.uint16, seed=9)
    conv = capi.DepthConverter(np.uint16, 1000.0)
    for normals in (False, True):
        for keep in (False, True):
            a = capi.depth_image_to_points(ctx, depth, ref.K_PINHOLE, conv, normals=normals, keep_invalid=keep,
                                           extrinsics=ref.pose(1))
            b = capi.depth_image_to_points(ctx, depth, ref.K_PINHOLE, conv, normals=normals, keep_invalid=keep,
                                           extrinsics=ref.pose(1), to_device=True)
            assert b["count"] == a["count"] == b["cloud"].n
            xyz, nrm = b["cloud"].download(normals=True) if normals else (b["cloud"].download(), None)
            assert np.array_equal(bits(xyz), bits(a["points"]))
            if normals:
                assert np.array_equal(bits(nrm), bits(a["normals"]))
            b["cloud"].close()


def render_points(seed, n=20000, w=64, h=48):
    """Points in front of, behind and beside the camera, at half-pixel projections, non-finite, out of the raw range,
    and many per pixel with exact raw-depth ties."""
    rng = np.random.default_rng(seed)
    z = rng.uniform(-0.5, 3.0, n)
    u = rng.uniform(-5, w + 5, n)
    v = rng.uniform(-5, h + 5, n)
    q = n // 10
    u[:q] = np.round(u[:q]) + 0.5
    z[:q] = 1.0
    z[q:2 * q] = np.round(z[q:2 * q] * 4) / 4
    u[q:2 * q] = np.round(u[q:2 * q] / 4)
    v[q:2 * q] = np.round(v[q:2 * q] / 4)
    p = np.stack([(u - w / 2) * z / 40.0, (v - h / 2) * z / 40.0, z], 1).astype(np.float32)
    p[-6:] = [[np.nan, 0, 1], [0, np.inf, 1], [0, 0, np.inf], [0, 0, 70.0], [0, 0, np.nan], [0, 0, -np.inf]]
    return p


def k_render(w, h):
    return np.array([[40.0, 0.0, w / 2], [0.0, 40.0, h / 2], [0.0, 0.0, 1.0]], np.float32)


@pytest.mark.parametrize("wh", [(1, 1), (1, 7), (7, 1), (2, 2), (3, 3), (64, 48), (640, 480)])
def test_rendering(ctx, wh):
    w, h = wh
    pts = render_points(w * h, w=w, h=h)
    col = np.random.default_rng(1).uniform(-0.2, 1.2, pts.shape).astype(np.float32)
    col[:50] = np.nan
    cloud = capi.Cloud(ctx, pts)
    for T in (None, ref.pose(4, angle=0.05, shift=0.05)):
        for K in (k_render(w, h), ref.K_GENERAL):
            want = ref.points_to_index_map(pts, K, w, h, T)
            assert np.array_equal(capi.points_to_index_map(ctx, pts, K, w, h, T), want)
            assert np.array_equal(capi.points_to_index_map(ctx, cloud, K, w, h, T), want)
            for dtype in DTYPES:
                for scale, md in ((1000.0, None), (1000.0, 2.0), (30000.0, None)):
                    conv = capi.DepthConverter(dtype, scale, md)
                    d = capi.points_to_depth_image(ctx, pts, K, w, h, conv, extrinsics=T)
                    assert np.array_equal(d.view(np.uint8), ref.points_to_depth_image(pts, K, w, h, dtype, scale, md,
                                                                                      None, T).view(np.uint8))
                    d2, rgb = capi.points_to_depth_image(ctx, cloud, K, w, h, conv, colors=col, extrinsics=T)
                    wd, wr = ref.points_to_depth_image(pts, K, w, h, dtype, scale, md, col, T)
                    assert np.array_equal(d2.view(np.uint8), wd.view(np.uint8)) and np.array_equal(rgb, wr)
    cloud.close()


def test_render_ties_pick_the_lowest_index(ctx):
    # 1000 points on one pixel with two raw depths: the first point of the nearer depth wins, with its colour
    pts = np.zeros((1000, 3), np.float32)
    pts[:, 2] = np.where(np.arange(1000) % 3 == 0, 1.25, 1.0)
    pts[:7, 2] = 1.25
    col = np.random.default_rng(0).uniform(0, 1, pts.shape).astype(np.float32)
    K = np.array([[10.0, 0, 1.0], [0, 10.0, 1.0], [0, 0, 1.0]], np.float32)
    d, rgb = capi.points_to_depth_image(ctx, pts, K, 3, 3, capi.DepthConverter(np.uint16, 1000.0), colors=col)
    assert d[1, 1] == 1000 and np.array_equal(rgb[1, 1], ref.color_bytes(col[7]))
    assert capi.points_to_index_map(ctx, pts, K, 3, 3)[1, 1] == 7


def test_launch_counts(ctx):
    depth = ref.frame("holed", 100, 80, np.uint16)
    conv = capi.DepthConverter(np.uint16, 1000.0)
    pts = render_points(0)
    for kw, launches in ((dict(keep_invalid=True), 1), (dict(keep_invalid=True, normals=True), 1),
                         (dict(), 5), (dict(normals=True), 5)):
        l0 = ctx.kernel_launches()
        capi.depth_image_to_points(ctx, depth, ref.K_PINHOLE, conv, **kw)
        assert ctx.kernel_launches() - l0 == launches, kw
    l0 = ctx.kernel_launches()
    capi.points_to_depth_image(ctx, pts, k_render(64, 48), 64, 48, conv)
    capi.points_to_index_map(ctx, pts, k_render(64, 48), 64, 48)
    assert ctx.kernel_launches() - l0 == 4


def test_no_device_memory_growth(ctx):
    import torch

    depth = ref.frame("holed", 640, 480, np.uint16)
    conv = capi.DepthConverter(np.uint16, 1000.0)
    pts = render_points(0)

    def once():
        r = capi.depth_image_to_points(ctx, depth, ref.K_PINHOLE, conv, normals=True, to_device=True)
        r["cloud"].close()
        capi.points_to_depth_image(ctx, pts, k_render(64, 48), 64, 48, conv, colors=np.ones_like(pts))
        capi.points_to_index_map(ctx, pts, k_render(64, 48), 64, 48)

    for _ in range(3):
        once()
    ctx.synchronize()
    free0 = torch.cuda.mem_get_info(0)[0]
    for _ in range(50):
        once()
    ctx.synchronize()
    assert free0 - torch.cuda.mem_get_info(0)[0] <= 8 << 20


def test_argument_errors(ctx):
    depth = np.ones((4, 4), np.uint16)
    lib = capi.lib()
    conv = capi.DepthConverter(np.uint16, 1000.0)
    K = ref.K_PINHOLE.reshape(9)
    cnt = capi.C.c_size_t()
    pts = np.empty((16, 3), np.float32)

    def back(depth_p=capi._p(depth), w=4, h=4, c=conv, K_p=capi._p(K), colors=None, normals=None, want_normals=0):
        return lib.cb_depth_image_to_points(ctx.h, depth_p, None, capi.C.c_size_t(w), capi.C.c_size_t(h),
                                            capi.C.byref(c) if c is not None else None, K_p, None,
                                            capi.C.c_int(want_normals), capi.C.c_int(0), capi._p(pts), normals, colors,
                                            capi.C.byref(cnt), None)

    assert back() == capi.CB_OK and cnt.value == 16
    assert back(depth_p=None) == -1
    assert back(K_p=None) == -1
    assert back(c=None) == -1
    assert back(w=0) == -1
    assert back(w=1 << 16, h=1 << 16) == -5
    assert back(c=capi.DepthConverter(np.uint16, 0.0)) == -1
    assert back(c=capi.DepthConverter(np.uint16, float("nan"))) == -1
    assert back(colors=capi._p(pts)) == -1  # colours without an rgb image
    assert back(normals=capi._p(pts)) == -1  # normals without want_normals
    bad = capi.DepthConverter(np.uint16, 1000.0)
    bad.raw_type = 7
    assert back(c=bad) == -1
    img = np.empty((4, 4), np.uint16)
    xyz = np.zeros((3, 3), np.float32)
    assert lib.cb_points_to_depth_image(ctx.h, None, None, capi.C.c_size_t(0), None, capi._p(K), None, capi.C.byref(conv),
                                        capi.C.c_size_t(4), capi.C.c_size_t(4), capi._p(img), None) == -1
    assert lib.cb_points_to_depth_image(ctx.h, capi._p(xyz), None, capi.C.c_size_t(3), capi._p(xyz), capi._p(K), None,
                                        capi.C.byref(conv), capi.C.c_size_t(4), capi.C.c_size_t(4), capi._p(img),
                                        None) == -1  # colours without an rgb output
    assert lib.cb_points_to_index_map(ctx.h, capi._p(xyz), None, capi.C.c_size_t(3), capi._p(K), None, capi.C.c_size_t(1 << 16),
                                      capi.C.c_size_t(1 << 16), capi._p(img)) == -5
    assert lib.cb_points_to_index_map(ctx.h, capi._p(xyz), None, capi.C.c_size_t(1 << 32), capi._p(K), None,
                                      capi.C.c_size_t(4), capi.C.c_size_t(4), capi._p(img)) == -5
    with pytest.raises(ValueError):
        capi.depth_image_to_points(ctx, depth.astype(np.float32), K, conv)


def scene(n=400000, seed=0):
    """A wall with relief, a floor and a box, 1.5-4 m in front of the camera, sampled densely."""
    rng = np.random.default_rng(seed)
    m = n // 3
    wall = np.stack([rng.uniform(-2, 2, m), rng.uniform(-1.5, 1.5, m), np.zeros(m)], 1)
    wall[:, 2] = 4.0 + 0.15 * np.sin(3 * wall[:, 0]) * np.cos(2 * wall[:, 1])
    floor = np.stack([rng.uniform(-2, 2, m), np.full(m, 1.0), rng.uniform(1.5, 4.0, m)], 1)
    a = rng.uniform(-0.4, 0.4, (m, 2))
    face = rng.integers(0, 3, m)
    box = np.zeros((m, 3))
    box[face == 0] = np.stack([a[face == 0, 0], a[face == 0, 1], np.full((face == 0).sum(), -0.4)], 1)
    box[face == 1] = np.stack([np.full((face == 1).sum(), -0.4), a[face == 1, 0], a[face == 1, 1]], 1)
    box[face == 2] = np.stack([a[face == 2, 0], np.full((face == 2).sum(), -0.4), a[face == 2, 1]], 1)
    box += [0.5, 0.4, 2.8]
    return np.concatenate([wall, floor, box]).astype(np.float32)


def test_two_pose_scene_registers(ctx):
    """Render the scene from two poses, convert both frames back with normals on the device, downsample, estimate
    normals and register with combined point-to-point / point-to-plane ICP: the pose is recovered within 2 mrad and
    5 mm."""
    w, h = 640, 480
    K = ref.K_PINHOLE
    pts = scene()
    TB = ref.pose(21, angle=0.01, shift=0.02)
    conv = capi.DepthConverter(np.uint16, 1000.0)
    clouds = []
    for T in (None, TB):
        d = capi.points_to_depth_image(ctx, pts, K, w, h, conv, extrinsics=T)
        c = capi.depth_image_to_points(ctx, d, K, conv, normals=True, to_device=True)["cloud"]
        ds = c.grid_downsample(0.02)
        ds.estimate_normals(k=10, fetch=False)
        clouds.append(ds)
    icp = capi.Icp(ctx, clouds[0], clouds[1])
    r = icp.estimate(metric="combined", w_pt=0.1, w_pl=1.0, max_iter=40, tol=1e-6, max_d2=0.1 ** 2)
    R, t = r["T"][:, :3].astype(np.float64), r["T"][:, 3].astype(np.float64)
    dR = R @ TB[:, :3].astype(np.float64).T
    ang = np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1))
    assert ang < 2e-3 and np.linalg.norm(t - TB[:, 3]) < 5e-3, (ang, t, TB[:, 3])


def test_index_map_of_a_cloud_adds_its_index_offset(ctx):
    pts = render_points(2)
    K = k_render(64, 48)
    want = capi.points_to_index_map(ctx, pts, K, 64, 48)
    cloud = capi.Cloud(ctx, pts, index_offset=1000)
    got = capi.points_to_index_map(ctx, cloud, K, 64, 48)
    empty = want == np.iinfo(np.uint64).max
    assert np.array_equal(got[empty], want[empty]) and np.array_equal(got[~empty], want[~empty] + 1000)
    cloud.close()


def test_device_frame_written_on_another_stream(ctx):
    """A frame a torch kernel is still writing on a side stream: the binding waits for the stream the array interface
    names before the library reads the frame."""
    torch = pytest.importorskip("torch")
    w, h = 1920, 1080
    depth = ref.frame("holed", w, h, np.float32, seed=8)
    want = capi.depth_image_to_points(ctx, depth, ref.K_PINHOLE, capi.DepthConverter(np.float32, 1000.0))
    src = torch.from_numpy(depth).cuda()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        dst = torch.zeros_like(src)
        for _ in range(20):  # keep the stream busy before the frame is written
            dst.copy_(torch.sin(src) * 0)
        dst.copy_(src)
        got = capi.depth_image_to_points(ctx, dst, ref.K_PINHOLE, capi.DepthConverter(np.float32, 1000.0))
    assert got["count"] == want["count"] and np.array_equal(bits(got["points"]), bits(want["points"]))
