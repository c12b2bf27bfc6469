"""Device memory ownership, measured: every buffer of the library except the context's IPC exchange region comes from
the device's default stream-ordered pool, so the pool's bytes in use (CU_MEMPOOL_ATTR_USED_MEM_CURRENT, read through
the driver API) show what the library holds. Once every entry point has run, running them all again must hold no
more memory, rejected inputs included; closing every object and then the context must return the pool to what it
held before the context existed."""
import ctypes as C
import gc

import numpy as np
import pytest

from cilantro_b200 import capi, synth

pytestmark = pytest.mark.gpu

CU_MEMPOOL_ATTR_USED_MEM_CURRENT = 7


@pytest.fixture(scope="module")
def pool_used():
    """Returns a function giving the bytes in use in device 0's default pool after a device-wide synchronise."""
    cu = C.CDLL("libcuda.so.1")

    def ok(rc, what):
        assert rc == 0, f"{what} failed with CUresult {rc}"

    ok(cu.cuInit(0), "cuInit")
    dev = C.c_int()
    ok(cu.cuDeviceGet(C.byref(dev), 0), "cuDeviceGet")
    pool = C.c_void_p()
    ok(cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev), "cuDeviceGetDefaultMemPool")
    pctx = C.c_void_p()
    ok(cu.cuDevicePrimaryCtxRetain(C.byref(pctx), dev), "cuDevicePrimaryCtxRetain")

    def used():
        ok(cu.cuCtxPushCurrent_v2(pctx), "cuCtxPushCurrent")
        try:
            ok(cu.cuCtxSynchronize(), "cuCtxSynchronize")
        finally:
            ok(cu.cuCtxPopCurrent_v2(C.byref(C.c_void_p())), "cuCtxPopCurrent")
        v = C.c_uint64()
        ok(cu.cuMemPoolGetAttribute(pool, C.c_int(CU_MEMPOOL_ATTR_USED_MEM_CURRENT), C.byref(v)),
           "cuMemPoolGetAttribute(USED_MEM_CURRENT)")
        return v.value

    yield used
    cu.cuDevicePrimaryCtxRelease_v2(dev)


def _rejected(fn):
    with pytest.raises(capi.CbError):
        fn()


def _every_entry_point(ctx, dst, src, icp, warp, warp_args, P):
    """Runs each entry point once; objects it creates are closed before it returns."""
    T = P["T"]
    capi.knn1_radius(ctx, dst, src, T, 1e-4)
    capi.knn_radius(ctx, dst, src, 8, T, 1e-2)
    capi.radius_search(ctx, dst, src, 1e-3, T)  # sizing call, then the fill
    capi.find_correspondences(ctx, dst, src, T, 1e-4)
    capi.transform_points(ctx, T, P["src"])
    nc = capi.Cloud(ctx, P["src"])
    nc.estimate_normals(k=10)
    nc.estimate_normals(radius2=0.05 ** 2)
    capi.grid_downsample(ctx, P["dst"], 0.05, normals=P["nrm"])
    down = dst.grid_downsample(0.05)
    down.close()
    nc.segment(k=10)
    nc.mean_shift(0.2, 5, 0.05, seeds=P["src"][:64])
    nc.close()
    a, b = capi.cloud_pair(ctx, P["dst"], P["nrm"], P["src"], None)
    a.close()
    b.close()
    rep = capi.Cloud.replicated(ctx, P["src"], None, 0, P["src"].shape[0])
    rep.close()
    cent = P["dst"][:5].copy()
    capi.kmeans_assign(ctx, dst, cent)
    capi.kmeans_cluster(ctx, dst, cent, max_iter=5)
    capi.ransac_score(ctx, dst, src, np.stack([T] * 3), 0.01)
    capi.ransac_rigid(ctx, dst, src, seed=1, max_iter=50, thresh=0.01)
    planes = np.array([[0, 0, 1, -0.5], [1, 0, 0, -0.5]], np.float32)
    capi.plane_score(ctx, dst, planes, 0.01)
    capi.ransac_plane(ctx, dst, seed=1, max_iter=50, thresh=0.01)
    capi.pca(ctx, dst)
    icp.estimate(max_iter=5)  # device-resident loop
    icp.estimate(max_iter=3, host_loop=True)
    icp.estimate(max_iter=3, search_dir="both")  # an engine mode
    icp.residuals(T)
    icp.correspondences()
    icp.accumulate(T)
    warp.estimate(max_iter=1, max_d2=0.04 ** 2)
    first, second, _ = warp.correspondences()
    warp.solve(first, second)
    m = warp_args[1].n
    warp.residuals(np.tile(np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32), (m, 1, 1)))
    # rejected inputs
    _rejected(lambda: capi.knn_radius(ctx, dst, src, 257))
    n = warp_args[1].n
    bad = (np.array([0, 2], np.uint64), np.array([0, n], np.int64), np.zeros(2, np.float32))
    _rejected(lambda: capi.WarpIcp(ctx, warp_args[0], warp_args[1], *bad))
    _rejected(lambda: dst.segment(k=257))
    _rejected(lambda: dst.estimate_normals(k=129))


def test_library_memory_returns_to_the_pool(pool_used):
    n = 4000
    d, s, nrm, T = synth.icp_pair(n, seed=7, noise=0.001, with_normals=True)
    P = dict(dst=d, src=s, nrm=nrm, T=T.astype(np.float32))
    W = synth.warp_pair(900, seed=5, spacing=0.005)
    gc.collect()
    gc.disable()
    try:
        before = pool_used()
        ctx = capi.Context(0)
        dst, src = capi.Cloud(ctx, d, nrm), capi.Cloud(ctx, s)
        icp = capi.Icp(ctx, dst, src)
        wdst, wsrc = capi.Cloud(ctx, W["dst"], W["dst_normals"]), capi.Cloud(ctx, W["src"])
        idx, d2, cnt = capi.knn_radius(ctx, wsrc, wsrc, 8)
        warp = capi.WarpIcp(ctx, wdst, wsrc, *capi.neighborhood_csr(idx, d2, cnt))
        _every_entry_point(ctx, dst, src, icp, warp, (wdst, wsrc), P)
        warm = pool_used()
        _every_entry_point(ctx, dst, src, icp, warp, (wdst, wsrc), P)
        again = pool_used()
        assert again == warm, f"a second round of calls holds {again - warm} more bytes"
        for obj in (warp, icp, wsrc, wdst, src, dst):
            obj.close()
        ctx.close()
        after = pool_used()
        assert after == before, f"{after - before} bytes still in use after the context was destroyed"
    finally:
        gc.enable()
