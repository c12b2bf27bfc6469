#!/usr/bin/env python
"""Small-size pass over every kernel family of libcilantro_b200.so: the target of scripts/sanitize.sh
(compute-sanitizer memcheck / racecheck / synccheck). Each call is checked against the oracle or a property, so a
sanitizer-clean run is also a correct run. Sizes are tiny: the sanitizers slow kernels down 10-1000x."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402
from cilantro_b200 import capi, synth  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
import kmeans_features_ref  # noqa: E402
import depth_images_ref  # noqa: E402
import pca_features_ref  # noqa: E402

N = int(os.environ.get("SANITIZE_N", "6000"))


def main():
    ctx = capi.Context(0)
    dst, src, nrm, T_ref = synth.icp_pair(N, seed=3, noise=0.002, with_normals=True)
    knn = oracle.BruteKnn(dst)
    d_dst, d_src = capi.Cloud(ctx, dst, nrm), capi.Cloud(ctx, src)
    max_d2 = np.float32(0.06 ** 2)
    # grid index + 1-NN kernel
    T = T_ref.astype(np.float32)
    idx, d2 = capi.knn1_radius(ctx, d_dst, d_src, T, max_d2)
    oi, od = knn.query(oracle.transform_points(T, src), max_d2)
    assert np.array_equal(idx, oi), "1-NN"
    icp = capi.Icp(ctx, d_dst, d_src)
    # device-resident loop (cold search kernel, cached pass with its searches, device solve) and host loop
    for kw in (dict(metric="p2p"), dict(metric="combined", w_pt=0.1, w_pl=1.0),
               dict(metric="combined", w_pt=0.1, w_pl=1.0, pt_rbf_sigma=0.01, pl_rbf_sigma=0.01)):
        want = oracle.icp(dst, src, knn, dst_n=nrm if kw["metric"] == "combined" else None, max_iter=5, tol=0.0, max_d2=max_d2, **kw)
        for host in (False, True):
            got = icp.estimate(max_iter=5, tol=0.0, max_d2=max_d2, host_loop=host, **kw)
            assert got["num_corr"] == want["num_corr"] and np.linalg.norm(got["T"].astype(np.float64) - want["T"]) < 1e-5, (kw, host)
    icp.estimate(metric="p2p", max_iter=4, tol=0.0, max_d2=max_d2)
    icp.loop_cache()
    icp.correspondences()
    icp.residuals(T, metric="combined", w_pt=0.1, w_pl=1.0)
    # inner Gauss-Newton iterations (stored correspondences) and the engine modes (pair lists, radix sorts)
    icp.estimate(metric="combined", w_pt=0.1, w_pl=1.0, max_iter=3, max_opt_iter=3, opt_tol=0.0, tol=0.0, max_d2=max_d2)
    for extra in (dict(search_dir="both", require_reciprocal=True), dict(inlier_fraction=0.7), dict(one_to_one=True),
                  dict(search_dir="first_to_second")):
        icp.estimate(metric="p2p", max_iter=2, tol=0.0, max_d2=max_d2, **extra)
        icp.correspondences()
    # feature-space search (feature_search.cu): both directions, one and two tails, the unbounded far sweep
    fs = synth.textured_sheet_pair(N, seed=4)
    ficp = capi.Icp(ctx, capi.Cloud(ctx, fs["dst"], fs["dst_normals"]), capi.Cloud(ctx, fs["src"]))
    for kind in ("point_color", "point_normal_color"):
        ficp.set_features(kind, dst_normals=fs["dst_normals"], dst_colors=fs["dst_colors"],
                          src_normals=fs["src_normals"], src_colors=fs["src_colors"], normal_weight=0.5, color_weight=5.0)
        for extra in (dict(), dict(search_dir="both")):
            ficp.estimate(metric="p2p", max_iter=2, tol=0.0, max_d2=max_d2, **extra)
            ficp.correspondences()
        ficp.estimate(metric="p2p", max_iter=1, tol=0.0, max_d2=np.float32(3e38), search_dir="first_to_second")
    ficp.set_features("point")
    ficp.close()
    # general-k kNN, radius lists, normals, downsample
    capi.knn_radius(ctx, d_dst, d_src, 8, T, np.float32(3e38))
    capi.radius_search(ctx, d_dst, d_src, np.float32(0.05 ** 2), T)
    sheet, _ = synth.surface_cloud(N, seed=5, noise=0.0005)
    c = capi.Cloud(ctx, sheet)
    ds = c.grid_downsample(0.03)
    ds.estimate_normals(k=8, view_point=[0.5, 0.5, 5.0])
    ds.estimate_normals(k=0, radius2=0.06 ** 2)
    # robust (MCD) normals: trials with refinements, kNN-in-radius, and the largest neighbourhood
    ds.estimate_normals_mcd(k=12, num_trials=2, num_refinements=1, chi_square_threshold=6.25, want_cov=True)
    ds.estimate_normals_mcd(k=16, radius2=0.06 ** 2, want_cov=True)
    ds.estimate_normals_mcd(k=128, inlier_ratio=0.5, min_sample_size=32)
    # connected-component segmentation: radius (all seeds, seed list) and kNN, with the normal / colour terms
    sheet_n = c.estimate_normals(k=8)["normals"]
    seg = capi.Cloud(ctx, sheet, sheet_n)
    seg.segment(radius2=0.02 ** 2, terms=capi.SEG_NORMALS, max_angle=0.2, min_size=3)
    seg.segment(radius2=0.02 ** 2, terms=capi.SEG_NORMALS | capi.SEG_COLORS, max_angle=-0.2, color_thresh=0.3,
                colors=np.abs(sheet_n), seeds=[0, 5, 5, N - 1])
    seg.segment(k=8, seeds=[3, 4])
    seg.segment(k=8, radius2=0.02 ** 2, max_size=50)
    # mean-shift: all points, a seed list with a far and a NaN seed, RBF weights, and many small batches
    ms = synth.mean_shift_scene(4, 200, sigma=0.05, seed=1)
    msc = capi.Cloud(ctx, ms["points"])
    msc.mean_shift(0.1, 20, 0.01)
    msc.mean_shift(0.1, 5, 0.01, seeds=np.concatenate([ms["points"][:50], [[9.0, 9.0, 9.0], [np.nan, 0.0, 0.0]]]))
    msc.mean_shift(0.1, 5, 0.01, weight=("rbf", 0.05))
    os.environ["CB_MEAN_SHIFT_PAIR_BUDGET"] = "500"
    msc.mean_shift(0.1, 3, 0.01)
    del os.environ["CB_MEAN_SHIFT_PAIR_BUDGET"]
    # k-means, RANSAC, PCA
    pts, cent = synth.kmeans_data(N, 16, seed=1)
    capi.kmeans_cluster(ctx, capi.Cloud(ctx, pts), cent, max_iter=3, tol=0.0)
    # D-dimensional k-means: partial dimension chunks and tiles, both sums paths, a repair, a NaN row
    rng = np.random.default_rng(4)
    for D, n, k in ((6, 1001, 3365), (17, 777, 129), (40, 300, 7)):
        rows = rng.standard_normal((n, D)).astype(np.float32)
        rows[5, D - 1] = np.nan
        c0 = np.vstack([rng.standard_normal((k - 1, D)), np.full((1, D), 50.0)]).astype(np.float32)
        v = capi.Vectors(ctx, rows)
        capi.kmeans_cluster(ctx, v, c0, max_iter=2, tol=0.0)
        assert np.array_equal(capi.kmeans_assign(ctx, v, c0)[0], kmeans_features_ref.assign(rows, c0)), ("k-means", D)
    rd, rs, _, _ = synth.ransac_pairs(N, 0.4, seed=2)
    c_rd, c_rs = capi.Cloud(ctx, rd), capi.Cloud(ctx, rs)
    capi.ransac_rigid(ctx, c_rd, c_rs, seed=5, max_iter=64, thresh=0.01)
    capi.pca(ctx, capi.Cloud(ctx, pts))
    # D-dimensional covariance / PCA: every column-tile width, partial chunks and tiles, a subset gather, a NaN value;
    # projection and reconstruction with partial row and output tiles
    for D, n in ((6, 1001), (13, 777), (31, 300), (70, 515)):
        rows = rng.standard_normal((n, D)).astype(np.float32)
        rows[5, D - 1] = np.nan
        v = capi.Vectors(ctx, rows)
        capi.pca(ctx, v, subset=np.arange(n)[::3])
        r = capi.pca(ctx, v)
        q = capi.pca_project(ctx, v, r["mean"], r["eigenvectors"], D // 2 + 1, to_device=True)
        capi.pca_reconstruct(ctx, q, r["mean"], r["eigenvectors"])
        np.testing.assert_array_equal(capi.pca_project(ctx, v, r["mean"], r["eigenvectors"], D),
                                      pca_features_ref.project(rows, r["mean"], r["eigenvectors"], D))
    # plane RANSAC: early exit with re-estimation, a full run of growing batches, tiny clouds, a NaN row
    ps = synth.plane_scene(N, seed=3)["points"]
    ps[7] = np.nan
    pc = capi.Cloud(ctx, ps)
    capi.ransac_plane(ctx, pc, 1, max_iter=250, thresh=0.01, inlier_count_thresh=N // 7)
    capi.ransac_plane(ctx, pc, 2, max_iter=300, thresh=0.01, inlier_count_thresh=N + 1, re_estimate=False)
    capi.plane_score(ctx, pc, np.tile([0.0, 0.0, 1.0, 0.0], (1100, 1)), 0.01)
    for m in (0, 1, 2, 3):
        capi.ransac_plane(ctx, capi.Cloud(ctx, ps[:m]), 4, max_iter=5)
    # dense warp-field ICP: assembly, the cooperative CG and compose over a few iterations, a solve with a fixed list,
    # residuals, and a NaN source point
    wp = synth.warp_pair(2000, seed=4)
    wp["src"][11] = np.nan
    wsrc = capi.Cloud(ctx, wp["src"])
    widx, wd2, wcnt = capi.knn_radius(ctx, wsrc, wsrc, 12)
    wicp = capi.WarpIcp(ctx, capi.Cloud(ctx, wp["dst"], wp["dst_normals"]), wsrc,
                        *capi.neighborhood_csr(widx, wd2, wcnt))
    got = wicp.estimate(w_pt=0.1, stiffness=200.0, huber=1e-2, reg_sigma=0.015, max_iter=3, max_d2=0.04 ** 2,
                        max_gn_iter=2, max_cg_iter=50)
    f, s, _ = wicp.correspondences()
    wicp.solve(f, s, w_pt=0.1, max_gn_iter=1, max_cg_iter=20)
    wicp.residuals(got["T"], w_pt=0.1)
    # sparse warp-field ICP: weights, resampling, assembly at points and nodes, the cooperative CG with its extra grid
    # sync and compose over the nodes; a duplicate node in one list, an empty list and a node nothing touches
    nodes = wsrc.grid_downsample(0.025)
    off, idx, val = capi.neighborhood_csr(*capi.knn_radius(ctx, nodes, wsrc, 4))
    cl = [list(idx[off[i]:off[i + 1]]) for i in range(len(off) - 1)]
    cv = [list(val[off[i]:off[i + 1]]) for i in range(len(off) - 1)]
    cl[3], cv[3] = cl[3] + cl[3][:1], cv[3] + cv[3][:1]
    cl[5], cv[5] = [], []
    coff = np.zeros(len(cl) + 1, np.uint64)
    coff[1:] = np.cumsum([len(a) for a in cl])
    ctrl = (coff, np.concatenate([np.asarray(a, np.int64) for a in cl]), np.concatenate([np.asarray(a, np.float32) for a in cv]))
    sicp = capi.SparseWarpIcp(ctx, capi.Cloud(ctx, wp["dst"], wp["dst_normals"]), wsrc, ctrl, nodes.n + 1,
                              capi.neighborhood_csr(*capi.knn_radius(ctx, nodes, nodes, 8)))
    got = sicp.estimate(stiffness=200.0, huber=1e-2, reg_sigma=0.075, ctrl_sigma=0.0125, max_iter=3,
                        max_d2=0.02 ** 2, max_gn_iter=2, max_cg_iter=50)
    f, s, _ = sicp.correspondences()
    sicp.solve(f, s, T_dense_src=got["T_dense"], max_gn_iter=1, max_cg_iter=20, ctrl_sigma=0.0125)
    sicp.resample(got["T"], ctrl_sigma=0.0125)
    sicp.residuals(got["T_dense"])
    # depth images: every back-projection pass (tile halo at the image edges, count / scan / write) and the z-buffer
    dimg = depth_images_ref.frame("holed", 45, 19, np.uint16)
    rgb = depth_images_ref.rgb_frame(45, 19)
    conv = capi.DepthConverter(np.uint16, 1000.0)
    for keep in (False, True):
        got = capi.depth_image_to_points(ctx, dimg, depth_images_ref.K_GENERAL, conv, rgb=rgb, normals=True,
                                         keep_invalid=keep)
        want = depth_images_ref.depth_to_points(dimg, depth_images_ref.K_GENERAL, 1000.0, None, rgb, None, True, keep)
        assert np.array_equal(got["points"], want[0], equal_nan=True), "depth image points"
    pts = got["points"]
    d, _ = capi.points_to_depth_image(ctx, pts, depth_images_ref.K_GENERAL, 45, 19, conv, colors=np.ones_like(pts))
    want = depth_images_ref.points_to_depth_image(pts, depth_images_ref.K_GENERAL, 45, 19, scale=1000.0)
    assert np.array_equal(d, want), "z-buffer"
    capi.points_to_index_map(ctx, pts, depth_images_ref.K_GENERAL, 45, 19)
    # projective ICP: the index map build, the per-query search (host loop, list path) and the device loop's pass
    moved = (pts + np.float32(0.002)).astype(np.float32)
    picp = capi.Icp(ctx, capi.Cloud(ctx, pts, got["normals"]), capi.Cloud(ctx, moved))
    picp.set_projection(depth_images_ref.K_GENERAL, 45, 19)
    for kw in (dict(metric="p2p"), dict(metric="combined", w_pt=0.1), dict(metric="combined", host_loop=True),
               dict(metric="p2p", inlier_fraction=0.5)):
        picp.estimate(max_iter=3, max_d2=np.float32(0.01), **kw)
    picp.correspondences()
    # projective warp-field ICPs: attach, estimate, re-attach, detach and estimate on the grid search
    pd, pm = capi.Cloud(ctx, pts, got["normals"]), capi.Cloud(ctx, moved)
    pnodes = pm.grid_downsample(0.05)
    for obj in (capi.WarpIcp(ctx, pd, pm, *capi.neighborhood_csr(*capi.knn_radius(ctx, pm, pm, 8))),
                capi.SparseWarpIcp(ctx, pd, pm, capi.neighborhood_csr(*capi.knn_radius(ctx, pnodes, pm, 4)), pnodes.n,
                                   capi.neighborhood_csr(*capi.knn_radius(ctx, pnodes, pnodes, 8)))):
        for K9, pw in ((depth_images_ref.K_GENERAL, 45), (depth_images_ref.K_GENERAL, 40), (None, 0)):
            obj.set_projection(K9, pw, 19 if K9 is not None else 0)
            obj.estimate(stiffness=200.0, huber=1e-2, max_iter=3, max_d2=np.float32(0.01), max_gn_iter=1,
                         max_cg_iter=30)
            obj.correspondences()
    ctx.close()
    print("sanitize target: all checks passed")


if __name__ == "__main__":
    main()
