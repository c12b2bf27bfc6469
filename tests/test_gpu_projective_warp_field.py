"""Projective correspondence search of the dense and sparse warp-field ICPs on the device (cb_warp_icp_set_projection,
cb_sparse_warp_icp_set_projection, DESIGN §4.22): correspondence lists bit for bit against the numpy fp32 restatement
of the search on the warped points, the whole loops against the fp32 and fp64 oracle loops searching through
ProjectiveKnn, detaching, launch counts, argument errors, device memory and a tracking run over rendered frames."""
import numpy as np
import pytest

import depth_images_ref as dimg
import icp_ref
import sparse_warp_field_ref as sref
from cilantro_b200 import capi, synth

pytestmark = pytest.mark.gpu

F = np.float32
ULP = 2.0 ** -24
EMPTY = np.iinfo(np.uint64).max
IDENTITY = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(F)
# the reference example's recipes (examples/non_rigid_icp.cpp): dense at a 5 mm spacing, sparse with 25 mm nodes
DENSE = dict(w_pt=0.1, w_pl=1.0, stiffness=200.0, huber=1e-2, max_gn_iter=1, gn_tol=5e-4, max_cg_iter=500, cg_tol=1e-5,
             reg_sigma=3 * 0.005)
DENSE_LOOP = dict(max_iter=15, tol=2.5e-3, max_d2=0.04 ** 2)
RES = 0.025
SPARSE = dict(w_pt=0.0, w_pl=1.0, stiffness=200.0, huber=1e-2, max_gn_iter=1, gn_tol=5e-4, max_cg_iter=500,
              cg_tol=1e-5, reg_sigma=3.0 * RES, ctrl_sigma=0.5 * RES)
SPARSE_LOOP = dict(max_iter=15, tol=2.5e-3, max_d2=0.02 ** 2)


class ProjectiveKnn:
    """The projective search as the oracle loops' knn: the warped points q are searched under the identity, as the
    device does (depth_images_ref's index map and projection, projective_ref's contract distance, kept iff < max_d2)."""

    def __init__(self, dst, K, w, h, E=None):
        self.dst, self.K, self.w, self.h, self.E = np.asarray(dst, F), K, w, h, E
        self.imap = dimg.points_to_index_map(dst, K, w, h, E).reshape(-1) if w * h else None

    def query(self, q, max_d2):
        n = q.shape[0]
        idx, d2 = np.full(n, -1, np.int64), np.full(n, F(max_d2), F)
        if self.imap is None or n == 0:
            return idx, d2
        p = icp_ref.apply_f32(IDENTITY, q)
        _, pix = dimg._project(p, self.K, self.E, self.w, self.h)
        s = np.nonzero(pix >= 0)[0]
        ind = self.imap[pix[s]]
        s, f = s[ind != EMPTY], ind[ind != EMPTY].astype(np.int64)
        with np.errstate(all="ignore"):
            d = p[s] - self.dst[f]
            v = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        keep = v < F(max_d2)
        idx[s[keep]], d2[s[keep]] = f[keep], v[keep]
        return idx, d2

    def list(self, q, max_d2):
        idx, d2 = self.query(q, max_d2)
        s = np.nonzero(idx >= 0)[0]
        return idx[s], s, d2[s]


@pytest.fixture(scope="module")
def wf(orc):
    from oracle import warp_field

    return warp_field


@pytest.fixture(scope="module")
def swf(orc):
    from oracle import sparse_warp_field

    return sparse_warp_field


def okw(kw):
    out = dict(kw)
    out["huber_delta"] = out.pop("huber")
    return out


def lift(P, E, depth=1.0):
    """P's clouds seen by a camera at pose E (world = E cam): the sheet centred on the optical axis at `depth`. K maps
    one mean point spacing to one pixel; the image is the sheet's extent plus a margin."""
    side, sp = P["side"], P["spacing"]
    c = np.array([side / 2, side / 2, -depth])
    R, t = np.asarray(E, np.float64)[:, :3], np.asarray(E, np.float64)[:, 3]
    out = dict(P)
    for k in ("dst", "src"):
        out[k] = ((P[k].astype(np.float64) - c) @ R.T + t).astype(F)
    out["dst_normals"] = (P["dst_normals"].astype(np.float64) @ R.T).astype(F)
    px = int(np.ceil(side / sp)) + 8
    f = depth / sp
    out["K"] = np.array([[f, 0, (px - 1) / 2], [0, f, (px - 1) / 2], [0, 0, 1]], F)
    out["w"] = out["h"] = px
    out["E"] = E
    return out


def k_for(w, h, side, depth, skew=False):
    """Intrinsics that spread a sheet of side `side` at `depth` over a w x h image; skewed with a general last row."""
    f = F(0.9 * max(min(w, h), 1) * depth / side)
    K = np.array([[f, 0, (w - 1) / 2], [0, f, (h - 1) / 2], [0, 0, 1]], F)
    if skew:
        K[0, 1], K[2] = F(0.02) * f, [0.001, -0.002, 1.25]
    return K


def dense_obj(ctx, dst, dst_n, src, nbhd=None):
    nb = nbhd if nbhd is not None else (np.zeros(1, np.uint64), np.zeros(0, np.int64), np.zeros(0, F))
    return capi.WarpIcp(ctx, capi.Cloud(ctx, dst, dst_n), capi.Cloud(ctx, src), *nb)


def sparse_obj(ctx, P):
    return capi.SparseWarpIcp(ctx, capi.Cloud(ctx, P["dst"], P["dst_normals"]), capi.Cloud(ctx, P["src"]), P["ctrl"],
                              P["m"], P["reg"])


def same_list(got, want):
    f, s, v = got
    wf_, ws, wv = want
    assert np.array_equal(f, wf_) and np.array_equal(s, ws), (f.size, wf_.size)
    assert np.array_equal(np.asarray(v, F).view(np.uint32), np.asarray(wv, F).view(np.uint32))


def list_scene(n, seed):
    """A sheet pair in front of the camera at the origin with exact destination duplicates (z ties) and a non-finite
    source point."""
    rng = np.random.default_rng(seed)
    P = synth.warp_pair(n, seed=seed, spacing=0.005)
    P = lift(P, IDENTITY)
    dup = rng.integers(0, n, max(1, n // 10))
    P["dst"] = np.vstack([P["dst"], P["dst"][dup]]).astype(F)
    P["dst_normals"] = np.vstack([P["dst_normals"], P["dst_normals"][dup]]).astype(F)
    P["src"] = np.vstack([P["src"], [[np.nan, 0.0, 1.0]]]).astype(F)
    return P


def general_transforms(n, seed, special=True):
    """Per-point transforms near the identity; with special rows that send their points behind the camera, far off
    the image, and a non-finite one."""
    rng = np.random.default_rng(seed)
    T = np.stack([dimg.pose(seed * 1000 + i, 0.01, 0.002) for i in range(min(n, 64))])
    T = np.ascontiguousarray(T[rng.integers(0, T.shape[0], n)])
    if special and n >= 4:
        T[0] = IDENTITY
        T[0, 2, 3] = -5.0  # behind the camera
        T[1] = IDENTITY
        T[1, 0, 3] = 40.0  # off the image
        T[2] = np.nan
    return T


@pytest.mark.parametrize("wh", [(1, 1), (31, 7), (640, 480), (1920, 1080)])
@pytest.mark.parametrize("general", [False, True])
def test_dense_lists_match_restatement(ctx, wf, wh, general):
    w, h = wh
    P = list_scene(20000 if w * h > 1000 else 3000, seed=w + 7 * general)
    E = dimg.pose(5, 0.05, 0.02) if general else None
    if general:  # the same scene seen from E: points and camera moved together
        P = dict(P, dst=icp_ref.apply_f32(E, P["dst"]), src=icp_ref.apply_f32(E, P["src"]))
    K = k_for(w, h, P["side"], 1.0, skew=general)
    n = P["src"].shape[0]
    T = general_transforms(n, seed=w)
    icp = dense_obj(ctx, P["dst"], P["dst_normals"], P["src"])
    icp.set_projection(K, w, h, E)
    knn = ProjectiveKnn(P["dst"], K, w, h, E)
    q = wf.apply(T, P["src"])
    inf_list = knn.list(q, F(np.inf))
    cuts = [F(1e-4), F(np.inf)]
    if inf_list[2].size:
        cuts.append(np.sort(inf_list[2])[inf_list[2].size // 2])  # values exactly at max_d2 are dropped
    for max_d2 in cuts:
        r = icp.estimate(T_init=T, **dict(DENSE, max_iter=1, max_d2=max_d2))
        want = knn.list(q, max_d2)
        same_list(icp.correspondences(), want)
        assert r["num_corr"] == want[0].size and r["iterations"] == 1
    assert inf_list[0].size > 0


def sparse_case(n, seed, E=IDENTITY):
    P = sref.make_case(n, RES, seed=seed)
    return lift(P, E)


@pytest.mark.parametrize("wh", [(1, 1), (31, 7), (640, 480), (1920, 1080)])
@pytest.mark.parametrize("general", [False, True])
def test_sparse_lists_match_restatement(ctx, wf, swf, wh, general):
    w, h = wh
    E = dimg.pose(6, 0.05, 0.02) if general else IDENTITY
    P = sparse_case(3000, seed=3 + w, E=E)
    # one point behind the camera and one off the image (they keep their control lists)
    P["src"] = P["src"].copy()
    P["src"][0] = icp_ref.apply_f32(E, np.array([[0.0, 0.0, -2.0]], F))[0]
    P["src"][1] = icp_ref.apply_f32(E, np.array([[30.0, 0.0, 1.0]], F))[0]
    K = k_for(w, h, P["side"], 1.0, skew=general)
    T = general_transforms(P["m"], seed=w, special=False)
    Td = swf.resample(T, P["ctrl"], P["m"], SPARSE["ctrl_sigma"])
    q = wf.apply(Td, P["src"])
    icp = sparse_obj(ctx, P)
    icp.set_projection(K, w, h, E if general else None)
    knn = ProjectiveKnn(P["dst"], K, w, h, E if general else None)
    for max_d2 in (F(1e-4), F(np.inf)):
        r = icp.estimate(T_init=T, **dict(SPARSE, max_iter=1, max_d2=max_d2))
        want = knn.list(q, max_d2)
        same_list(icp.correspondences(), want)
        assert r["num_corr"] == want[0].size


def test_empty_images_give_no_correspondences(ctx):
    P = list_scene(500, seed=2)
    K = k_for(64, 48, P["side"], 1.0)
    icp = dense_obj(ctx, P["dst"], P["dst_normals"], P["src"])
    for w, h in ((0, 48), (64, 0), (0, 0)):
        icp.set_projection(K, w, h)
        r = icp.estimate(**dict(DENSE, max_iter=3))
        assert r["num_corr"] == 0 and r["iterations"] == 1 and r["last_delta"] == 0.0
        assert np.array_equal(r["T"], np.tile(IDENTITY, (P["src"].shape[0], 1, 1)))
        assert icp.correspondences()[0].size == 0


def loop_check(got, o32, o64, src, side, apply):
    assert got["iterations"] == o32["iterations"]
    assert got["converged"] == o32["converged"]
    key = "T_dense" if "T_dense" in got else "T"
    q_dev, q32, q64 = (apply(r[key], src) for r in (got, o32, o64))
    spread = np.abs(q32 - q64).max()
    err = np.abs(q_dev - q32).max()
    assert err <= 4 * spread + 16 * ULP * side, (err, spread)
    assert abs(got["num_corr"] - o32["num_corr"]) <= max(2 * abs(o32["num_corr"] - o64["num_corr"]), 2)


def test_dense_loop_against_oracles(ctx, orc, wf):
    P = lift(synth.warp_pair(2000, seed=3, spacing=0.005), dimg.pose(8, 0.1, 0.05))
    idx, d2, cnt = orc.BruteKnn(P["src"]).neighborhoods(P["src"], 12, 3.0e38)
    nb = capi.neighborhood_csr(idx, d2, cnt)
    icp = dense_obj(ctx, P["dst"], P["dst_normals"], P["src"], nb)
    icp.set_projection(P["K"], P["w"], P["h"], P["E"])
    got = icp.estimate(**DENSE, **DENSE_LOOP)
    knn = ProjectiveKnn(P["dst"], P["K"], P["w"], P["h"], P["E"])
    o32 = wf.icp(P["dst"], P["dst_normals"], P["src"], nb, knn=knn, **DENSE_LOOP, **okw(DENSE))
    o64 = wf.icp(P["dst"], P["dst_normals"], P["src"], nb, knn=knn, double=True, **DENSE_LOOP, **okw(DENSE))
    loop_check(got, o32, o64, P["src"], P["side"], wf.apply)
    assert got["iterations"] > 1 and got["num_corr"] > 1000
    # residuals stay the kd-tree search: those of the kd-tree object, bit for bit
    kd = dense_obj(ctx, P["dst"], P["dst_normals"], P["src"], nb)
    kw = {k: DENSE[k] for k in ("w_pt", "w_pl")}
    assert np.array_equal(icp.residuals(got["T"], **kw).view(np.uint32), kd.residuals(got["T"], **kw).view(np.uint32))


@pytest.mark.parametrize("big", [False, True])
def test_sparse_loop_against_oracles(ctx, orc, wf, swf, big):
    # big: more source points than the cooperative CG grid has threads (every grid-stride loop wraps)
    n = int(1.1 * 2048 * ctx.device_info()["sm_count"]) + 1000 if big else 4000
    P = sparse_case(n, seed=6, E=dimg.pose(9, 0.1, 0.05))
    icp = sparse_obj(ctx, P)
    icp.set_projection(P["K"], P["w"], P["h"], P["E"])
    got = icp.estimate(**SPARSE, **SPARSE_LOOP)
    knn = ProjectiveKnn(P["dst"], P["K"], P["w"], P["h"], P["E"])
    args = (P["dst"], P["dst_normals"], P["src"], P["ctrl"], P["m"], P["reg"])
    o32 = swf.icp(*args, knn=knn, **SPARSE_LOOP, **okw(SPARSE))
    o64 = swf.icp(*args, knn=knn, double=True, **SPARSE_LOOP, **okw(SPARSE))
    loop_check(got, o32, o64, P["src"], P["side"], wf.apply)
    assert got["iterations"] > 1 and got["num_corr"] > n // 4
    kd = sparse_obj(ctx, P)
    kw = {k: SPARSE[k] for k in ("w_pt", "w_pl")}
    assert np.array_equal(icp.residuals(got["T_dense"], **kw).view(np.uint32),
                          kd.residuals(got["T_dense"], **kw).view(np.uint32))


def test_detach_restores_the_grid_search(ctx, wf):
    P = sparse_case(3000, seed=4)
    icp, fresh = sparse_obj(ctx, P), sparse_obj(ctx, P)
    icp.set_projection(P["K"], P["w"], P["h"])
    proj = icp.estimate(**SPARSE, **SPARSE_LOOP)
    icp.set_projection(None, 0, 0)
    with pytest.raises(capi.CbError, match="error -1"):
        icp.correspondences()
    a, b = icp.estimate(**SPARSE, **SPARSE_LOOP), fresh.estimate(**SPARSE, **SPARSE_LOOP)
    for k in ("T", "T_dense"):
        assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32))
    assert (a["iterations"], a["num_corr"], a["cg_iterations"]) == (b["iterations"], b["num_corr"], b["cg_iterations"])
    la, lb = icp.correspondences(), fresh.correspondences()
    same_list(la, lb)
    # re-attaching with another K rebuilds the map: the run is the projective one of that K
    K2 = P["K"].copy()
    K2[0, 2] += 3.0
    icp.set_projection(P["K"], P["w"], P["h"])
    again = icp.estimate(**SPARSE, **SPARSE_LOOP)
    assert np.array_equal(again["T"].view(np.uint32), proj["T"].view(np.uint32))
    icp.set_projection(K2, P["w"], P["h"])
    with pytest.raises(capi.CbError, match="error -1"):
        icp.correspondences()
    other = icp.estimate(**dict(SPARSE, max_iter=1, max_d2=SPARSE_LOOP["max_d2"]))
    Td = icp.resample(np.tile(IDENTITY, (P["m"], 1, 1)), ctrl_sigma=SPARSE["ctrl_sigma"])
    want = ProjectiveKnn(P["dst"], K2, P["w"], P["h"]).list(wf.apply(Td, P["src"]), F(SPARSE_LOOP["max_d2"]))
    same_list(icp.correspondences(), want)
    assert other["num_corr"] == want[0].size
    # dense: detach then estimate equals a fresh object
    d1, d2 = dense_obj(ctx, P["dst"], P["dst_normals"], P["src"]), dense_obj(ctx, P["dst"], P["dst_normals"], P["src"])
    d1.set_projection(P["K"], P["w"], P["h"])
    d1.estimate(**dict(DENSE, max_iter=2))
    d1.set_projection(None, 0, 0)
    x, y = d1.estimate(**dict(DENSE, max_iter=3)), d2.estimate(**dict(DENSE, max_iter=3))
    assert np.array_equal(x["T"].view(np.uint32), y["T"].view(np.uint32)) and x["num_corr"] == y["num_corr"]
    same_list(d1.correspondences(), d2.correspondences())


def test_launch_counts(ctx, orc):
    P = sparse_case(3000, seed=5)
    kw = dict(SPARSE, max_iter=3, tol=0.0, max_d2=SPARSE_LOOP["max_d2"], cg_tol=0.0)
    proj, kd = sparse_obj(ctx, P), sparse_obj(ctx, P)
    proj.set_projection(P["K"], P["w"], P["h"])
    a = proj.estimate(**dict(kw, max_cg_iter=10))
    b = proj.estimate(**dict(kw, max_cg_iter=200))
    c = kd.estimate(**dict(kw, max_cg_iter=10))
    assert a["iterations"] == c["iterations"] == 3 and a["gn_steps"] == c["gn_steps"] == 3
    assert a["kernel_launches"] == b["kernel_launches"] == c["kernel_launches"]
    again = proj.estimate(**dict(kw, max_cg_iter=10))
    for k in ("T", "T_dense"):
        assert np.array_equal(a[k].view(np.uint32), again[k].view(np.uint32))
    dn, dk = (dense_obj(ctx, P["dst"], P["dst_normals"], P["src"]) for _ in range(2))
    dn.set_projection(P["K"], P["w"], P["h"])
    kw = dict(DENSE, max_iter=3, tol=0.0, cg_tol=0.0)
    x, y, z = (o.estimate(**dict(kw, max_cg_iter=m)) for o, m in ((dn, 10), (dn, 200), (dk, 10)))
    assert x["gn_steps"] == z["gn_steps"] == 3
    assert x["kernel_launches"] == y["kernel_launches"] == z["kernel_launches"]


def test_argument_errors_keep_the_attached_map(ctx, orc):
    P = sparse_case(3000, seed=7)
    for icp, est in ((sparse_obj(ctx, P), SPARSE), (dense_obj(ctx, P["dst"], P["dst_normals"], P["src"]), DENSE)):
        icp.set_projection(P["K"], P["w"], P["h"])
        want = icp.estimate(**dict(est, max_iter=2))
        bad = P["K"].copy()
        bad[1, 1] = np.nan
        for args in ((bad, P["w"], P["h"], None), (P["K"], P["w"], P["h"], np.full((3, 4), np.inf, F)),
                     (P["K"], 1 << 16, 1 << 16, None)):
            with pytest.raises(capi.CbError, match="error -1"):
                icp.set_projection(*args)
        got = icp.estimate(**dict(est, max_iter=2))
        assert np.array_equal(got["T"].view(np.uint32), want["T"].view(np.uint32))
        assert got["num_corr"] == want["num_corr"]
        for kw in (dict(inlier_fraction=0.5), dict(search_dir="both"), dict(one_to_one=True),
                   dict(require_reciprocal=True)):
            with pytest.raises(capi.CbError, match="error -5"):
                icp.estimate(**dict(est, max_iter=2, **kw))


def test_no_device_memory_growth(ctx, orc):
    import torch

    P = sparse_case(3000, seed=8)
    icp = sparse_obj(ctx, P)
    dc, sc = capi.Cloud(ctx, P["dst"], P["dst_normals"]), capi.Cloud(ctx, P["src"])
    nb = (np.zeros(1, np.uint64), np.zeros(0, np.int64), np.zeros(0, F))
    for _ in range(3):
        icp.set_projection(P["K"], P["w"], P["h"])
        icp.estimate(**dict(SPARSE, max_iter=3))
    ctx.synchronize()
    free0 = torch.cuda.mem_get_info(0)[0]
    for k in range(20):
        icp.set_projection(P["K"], P["w"] + k % 3, P["h"])
        icp.estimate(**dict(SPARSE, max_iter=3))
        o = capi.WarpIcp(ctx, dc, sc, *nb)
        o.set_projection(P["K"], P["w"], P["h"])
        o.estimate(**dict(DENSE, max_iter=2))
        o.close()
    ctx.synchronize()
    assert free0 - torch.cuda.mem_get_info(0)[0] <= 8 << 20


def sheet(k, n=900):
    """Frame k of a deforming sheet (0.8 x 0.6 m, 1 m in front of the camera): a fixed relief plus a bend that grows
    with k; n x n samples, far more than the rendered pixels."""
    x, y = np.meshgrid(np.linspace(-0.4, 0.4, n), np.linspace(-0.3, 0.3, n))
    z = 1.0 + 0.02 * np.sin(6 * x) * np.cos(5 * y) + 0.004 * k * (x / 0.4) ** 2 - 0.002 * k * (y / 0.3)
    return np.stack([x, y, z], -1).reshape(-1, 3).astype(F)


def test_tracking_rendered_deforming_frames(ctx, orc):
    """Every frame of a bending sheet, rendered at 640 x 480 and converted back with normals on the device, tracked
    against the first frame with the sparse projective object and the reference example's recipe."""
    w, h = 640, 480
    K = np.array([[525, 0, 319.5], [0, 525, 239.5], [0, 0, 1]], F)
    conv = capi.DepthConverter(np.float32, 1.0)

    def frame(k):
        depth = capi.points_to_depth_image(ctx, sheet(k), K, w, h, conv)
        r = capi.depth_image_to_points(ctx, depth, K, conv, normals=True)
        return r["points"], r["normals"]

    dst, dst_n = frame(0)
    model = capi.Cloud(ctx, dst, dst_n)
    for k in range(1, 5):
        src, _ = frame(k)
        nodes, _, _ = orc.grid_downsample(src, RES)
        knn = orc.BruteKnn(nodes)
        ctrl = capi.neighborhood_csr(*knn.neighborhoods(src, 4, 3.0e38))
        reg = capi.neighborhood_csr(*knn.neighborhoods(nodes, 8, 3.0e38))
        icp = capi.SparseWarpIcp(ctx, model, capi.Cloud(ctx, src), ctrl, nodes.shape[0], reg)
        icp.set_projection(K, w, h)
        r = icp.estimate(**SPARSE, **SPARSE_LOOP)
        kw = dict(w_pt=0.0, w_pl=1.0)
        before = icp.residuals(np.tile(IDENTITY, (src.shape[0], 1, 1)), **kw).mean()
        after = icp.residuals(r["T_dense"], **kw).mean()
        print(f"frame {k}: {r['iterations']} iterations, {r['num_corr']} correspondences, "
              f"residual {before:.3e} -> {after:.3e}")
        assert after < 0.5 * before, (k, before, after)
