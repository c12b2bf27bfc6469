"""Secondary workloads of bench.py (BASELINE.json configs 4 and 5, and PCA): single GPU, one JSON line each.

    python bench.py --workload kmeans_50m   [--steps K --warmup W]     step = one Lloyd iteration
    python bench.py --workload ransac_5m    [--steps K --warmup W]     step = one batch of 1000 hypotheses
    python bench.py --workload pca_50m      [--steps K --warmup W]     step = one mean+covariance pass
    python bench.py --workload segment_1m   [--steps K --warmup W]     step = one all-seeds segmentation (radius)
    python bench.py --workload segment_knn_1m                           step = one all-seeds segmentation (kNN 10)
    python bench.py --workload meanshift_1m [--steps K --warmup W]     step = one all-seeds mean-shift call
    python bench.py --workload ransac_plane_5m [--steps K --warmup W]  step = one batch of 1000 plane hypotheses

Same timing hygiene as the ICP workload (CUDA events inside the library, inputs larger than L2 or an L2
flush, CPU baseline = the oracle on a bounded sample of the same workload).
"""
import json
import time

import numpy as np

FP32_PEAK_TFLOPS = 132 * 128 * 2 * 1.98e9 / 1e12  # H100 SXM nominal FMA rate of the FP32 pipe (SMs x lanes x 2 x max clock)


def _ctx(ctx=None):
    import torch

    from cilantro_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("bench needs a CUDA device: cilantro_b200 has no CPU fallback")
    return capi, (ctx if ctx is not None else capi.Context(0))


def brief(line):
    """The fields of a workload line that bench.py's `secondary` block carries."""
    keep = ("metric", "value", "unit", "iterations_per_sec", "n_gpus", "steps", "warmup", "ms_per_step", "scaling", "dtype",
            "config", "e2e", "gpu_launches", "roofline", "cpu_baseline", "parity")
    return {k: line[k] for k in keep if k in line}


def kmeans(args, n=50_000_000, k=1024, ctx=None, rank=0, world=1):
    """KMeans3f, BASELINE config 4. world > 1: the points are split into contiguous shards, one per rank (all ranks
    call this; the library all-reduces the K x 4 centroid sums per iteration); rank 0 returns the line."""
    import oracle
    from cilantro_b200 import synth
    from cilantro_b200.dist import max_over_ranks, shard_bounds

    capi, ctx = _ctx(ctx)
    pts, cent0 = synth.kmeans_data(n, k, seed=1)
    lo, hi = shard_bounds(n, rank, world)
    mine = np.ascontiguousarray(pts[lo:hi])
    cloud = capi.Cloud(ctx, mine, None, index_offset=lo)
    # warm-up
    capi.kmeans_cluster(ctx, cloud, cent0, max_iter=max(args.warmup, 1), tol=0.0, want_labels=False)
    l0 = ctx.kernel_launches()
    res = capi.kmeans_cluster(ctx, cloud, cent0, max_iter=args.steps, tol=0.0, want_labels=False)
    launches = ctx.kernel_launches() - l0
    ms = max_over_ranks(res["gpu_ms_total"]) / res["iterations"]
    flop = 8.0 * n * k
    # e2e: host points -> upload -> cluster(steps) -> centroids + labels on host
    t0 = time.perf_counter()
    c2 = capi.Cloud(ctx, mine, None, index_offset=lo)
    r2 = capi.kmeans_cluster(ctx, c2, cent0, max_iter=args.steps, tol=0.0, want_labels=True)
    e2e_s = max_over_ranks(time.perf_counter() - t0)
    c2.close()
    cloud.close()
    if rank != 0:
        return None
    # CPU baseline + parity: the oracle's assignment step (OpenMP) on a bounded sample; labels must be bit-exact
    sample = min(hi - lo, 2_000_000)
    t0 = time.perf_counter()
    oc = oracle.kmeans(pts[:sample], cent0, max_iter=1, tol=0.0)
    cpu_s = time.perf_counter() - t0
    parity = None
    if world == 1:  # (with several ranks every clustering call on ctx is a collective)
        c3 = capi.Cloud(ctx, np.ascontiguousarray(pts[:sample]))
        g1 = capi.kmeans_cluster(ctx, c3, cent0, max_iter=1, tol=0.0, want_labels=True)
        c3.close()
        parity = {"labels_equal_after_one_iteration": bool(np.array_equal(g1["labels"], oc[1])), "points": int(sample),
                  "centroid_max_abs_diff": float(np.abs(g1["centroids"] - oc[0]).max())}
    line = {
        "metric": "kmeans_point_assignments_per_sec", "value": n * 1e3 / ms, "unit": "points/s",
        "iterations_per_sec": 1e3 / ms, "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms,
        "higher_is_better": True, "scaling": "strong" if world > 1 else "weak", "vs_baseline": None, "dtype": "f32",
        "data": "synthetic",
        "config": {"workload": f"KMeans3f: {n} uniform points ({hi - lo} per GPU x {world}), K={k}, fixed initial centroids, "
                               f"{args.steps} Lloyd iterations (tol=0)",
                   "parallelism": f"points sharded x{world}, centroids replicated, one ncclAllReduce of K x 4 doubles per iteration",
                   "l2": "inputs (600 MB) larger than L2"},
        "e2e": {"value": n * args.steps / e2e_s, "unit": "points/s", "h2d_bytes_per_step": mine.nbytes / args.steps,
                "d2h_bytes_per_step": (8 * (hi - lo) + 12 * k) / args.steps,
                "what": f"cb_cloud_create + cb_kmeans_cluster({args.steps}) + labels/centroids on host: {e2e_s:.3f} s"},
        "gpu_launches": int(launches),
        "roofline": {"bound": "fp32", "achieved": flop / (ms * 1e-3) / 1e12 / world, "peak": FP32_PEAK_TFLOPS, "unit": "TFLOP/s",
                     "frac": flop / (ms * 1e-3) / 1e12 / world / FP32_PEAK_TFLOPS, "traffic": None,
                     "kernel": "kmeans_assign_kernel", "peak_source": "nominal: 132 SMs x 128 lanes x 2 x 1.98 GHz (H100 SXM)",
                     "note": "per GPU; 8 N K flop per iteration (3 sub, 3 mul, 2 add; the "
                     "arithmetic contract forbids FMA, so the attainable rate is half the FMA peak)"},
        "cpu_baseline": {"value": sample / cpu_s, "unit": "points/s", "cores": oracle.num_threads(), "kind": "port",
                         "sample": f"1 Lloyd iteration on the first {sample} points (brute-force assignment, OpenMP; serial update)"},
        "parity": parity,
    }
    return line


def ransac(args, n=5_000_000, batch=1000, ctx=None):
    import oracle
    from cilantro_b200 import synth

    capi, ctx = _ctx(ctx)
    dst, src, T_ref, inl = synth.ransac_pairs(n, 0.3, seed=1)
    d_dst, d_src = capi.Cloud(ctx, dst), capi.Cloud(ctx, src)
    # hypotheses: the generating pose plus random rigid perturbations of it (inputs of the measured scoring call;
    # the oracle below only scores a few of them as the CPU baseline / checker)
    rng = np.random.default_rng(7)
    T_h = np.empty((batch, 3, 4), np.float32)
    T_h[0] = T_ref.astype(np.float32)
    R0, t0_ = np.asarray(T_ref)[:, :3], np.asarray(T_ref)[:, 3]
    for h in range(1, batch):
        dT = np.asarray(synth.rigid_from_axis_angle(rng.standard_normal(3), 0.05 * rng.standard_normal(),
                                                    0.05 * rng.standard_normal(3)))
        T_h[h] = np.hstack([dT[:, :3] @ R0, (dT[:, :3] @ t0_ + dT[:, 3])[:, None]]).astype(np.float32)
    for _ in range(max(args.warmup, 1)):
        capi.ransac_score(ctx, d_dst, d_src, T_h[:64], 0.01)
    l0 = ctx.kernel_launches()
    times = []
    for _ in range(args.steps):
        ctx.synchronize()
        t0 = time.perf_counter()
        counts = capi.ransac_score(ctx, d_dst, d_src, T_h, 0.01)
        times.append(time.perf_counter() - t0)
    launches = ctx.kernel_launches() - l0
    ms = 1e3 * float(np.median(times))
    flop = 30.0 * n * batch
    # full loop, 10k hypotheses, early exit disabled (BASELINE config 5)
    t0 = time.perf_counter()
    full = capi.ransac_rigid(ctx, d_dst, d_src, seed=11, max_iter=10000, thresh=0.01, inlier_count_thresh=n,
                             re_estimate=True)
    full_s = time.perf_counter() - t0
    err = synth.frobenius(full["T"], T_ref)
    hyp_cpu = 8
    t0 = time.perf_counter()
    oc = oracle.ransac_score(dst, src, T_h[:hyp_cpu], 0.01)
    cpu_s = time.perf_counter() - t0
    assert np.array_equal(oc, counts[:hyp_cpu]), "GPU inlier counts differ from the oracle"
    line = {
        "metric": "ransac_hypotheses_per_sec", "value": batch * 1e3 / ms, "unit": "hypotheses/s", "n_gpus": 1,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": f"RigidTransformRANSACEstimator3f scoring: {n} correspondences (30 % inliers), {batch} hypotheses per step, thresh 0.01",
                   "l2": "inputs (120 MB) larger than L2; the pairs are read once per batch"},
        "e2e": {"value": full["iterations"] / full_s, "unit": "hypotheses/s", "h2d_bytes_per_step": 48.0 * 1000, "d2h_bytes_per_step": 4.0 * 1000,
                "what": f"cb_ransac_rigid: 10000 hypotheses (sample on host, Kabsch-of-3 on host, batches of 1024 scored on the "
                        f"device, re-estimation) in {full_s:.3f} s; |T - T_ref|_F = {err:.2e}; inliers {full['num_inliers']}"},
        "gpu_launches": int(launches),
        "roofline": {"bound": "fp32", "achieved": flop / (ms * 1e-3) / 1e12, "peak": FP32_PEAK_TFLOPS, "unit": "TFLOP/s",
                     "frac": flop / (ms * 1e-3) / 1e12 / FP32_PEAK_TFLOPS, "traffic": None, "kernel": "ransac_score_kernel",
                     "note": "~30 flop per pair-hypothesis (SURVEY 8d), no FMA by contract; wall-clock per call incl. 48 KB H2D + 4 KB D2H"},
        "cpu_baseline": {"value": hyp_cpu / cpu_s, "unit": "hypotheses/s", "cores": oracle.num_threads(), "kind": "port",
                         "sample": f"{hyp_cpu} hypotheses scored over all {n} pairs (OpenMP over hypotheses)"},
        "parity": {"inlier_counts_equal": True, "hypotheses_compared": hyp_cpu, "pairs": n},
    }
    return line


def pca(args, n=50_000_000, ctx=None):
    import oracle
    from cilantro_b200 import synth

    capi, ctx = _ctx(ctx)
    pts, _ = synth.kmeans_data(n, 1, seed=2)
    cloud = capi.Cloud(ctx, pts)
    for _ in range(max(args.warmup, 1)):
        capi.pca(ctx, cloud)
    times = []
    l0 = ctx.kernel_launches()
    for _ in range(args.steps):
        ctx.synchronize()
        t0 = time.perf_counter()
        r = capi.pca(ctx, cloud)
        times.append(time.perf_counter() - t0)
    launches = ctx.kernel_launches() - l0
    ms = 1e3 * float(np.median(times))
    from bench import load_peaks

    peak, src = load_peaks()
    sample = 10_000_000
    t0 = time.perf_counter()
    o = oracle.pca(pts[:sample])
    cpu_s = time.perf_counter() - t0
    # parity on the CPU sample: the same points through the device path
    cs = capi.Cloud(ctx, np.ascontiguousarray(pts[:sample]))
    g = capi.pca(ctx, cs)
    cs.close()
    pca_parity = _pca_parity(g, o, sample)
    line = {
        "metric": "pca_points_per_sec", "value": n * 1e3 / ms, "unit": "points/s", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f64 accumulation of f32 points", "data": "synthetic",
        "config": {"workload": f"PrincipalComponentAnalysis3f: {n} uniform points (mean + covariance + 3x3 eigen)",
                   "l2": "inputs (600 MB) larger than L2"},
        "e2e": {"value": None, "unit": "points/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 80,
                "what": "wall clock per cb_pca call on a resident cloud (pivot launch + streaming pass + host eigen-solve)"},
        "gpu_launches": int(launches),
        "roofline": {"bound": "hbm", "achieved": 12.0 * n / (ms * 1e-3) / 1e9, "peak": peak, "unit": "GB/s",
                     "frac": 12.0 * n / (ms * 1e-3) / 1e9 / peak, "traffic": None, "kernel": "moments_kernel", "peak_source": src},
        "cpu_baseline": {"value": sample / cpu_s, "unit": "points/s", "cores": 1, "kind": "port",
                         "sample": f"serial two-pass covariance (the reference's default, covariance.hpp:64-76) on {sample} points"},
        "parity": pca_parity,
    }
    return line


def normals(args, n=5_000_000, k=10, ctx=None):
    """PointCloud3f::estimateNormalsKNN(k) (view point = origin) on a synthetic scanned sheet."""
    import oracle
    from cilantro_b200 import synth
    from bench import load_peaks

    capi, ctx = _ctx(ctx)
    pts, _ = synth.surface_cloud(n, seed=1, noise=0.0005)
    cloud = capi.Cloud(ctx, pts)
    vp = [0.0, 0.0, 0.0]
    for _ in range(max(args.warmup, 1)):
        cloud.estimate_normals(k=k, view_point=vp, fetch=False)
    l0 = ctx.kernel_launches()
    ms_list = []
    for _ in range(args.steps):
        ctx.flush_l2()
        ms_list.append(cloud.estimate_normals(k=k, view_point=vp, fetch=False)["gpu_ms"])
    launches = ctx.kernel_launches() - l0
    ms = float(np.mean(ms_list))
    # e2e: host points -> upload -> grid -> normals -> normals on host
    e2e = []
    for _ in range(3):
        t0 = time.perf_counter()
        c2 = capi.Cloud(ctx, pts)
        c2.estimate_normals(k=k, view_point=vp, want_curvature=False)
        e2e.append(time.perf_counter() - t0)
        c2.close()
    e2e_s = min(e2e)
    peak, src = load_peaks()
    sample = min(n, 2_000_000)
    knn = oracle.make_knn(pts[:sample])
    t0 = time.perf_counter()
    oracle.estimate_normals(pts[:sample], knn, k=k, view_point=vp)
    cpu_s = time.perf_counter() - t0
    algo = 28.0 * n  # read float4 point once + write one 12 B normal (the cell-sorted float4 copy is internal)
    line = {
        "metric": "normal_estimation_points_per_sec", "value": n * 1e3 / ms, "unit": "points/s", "n_gpus": 1,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": f"PointCloud3f::estimateNormalsKNN({k}) on a {n}-point noisy sheet, view point = origin",
                   "l2": "flushed before every timed call"},
        "e2e": {"value": n / e2e_s, "unit": "points/s", "h2d_bytes_per_step": pts.nbytes, "d2h_bytes_per_step": 12 * n,
                "what": f"cb_cloud_create + cb_cloud_estimate_normals + normals on host: {e2e_s * 1e3:.1f} ms"},
        "gpu_launches": int(launches),
        "roofline": {"bound": "hbm", "achieved": algo / (ms * 1e-3) / 1e9, "peak": peak, "unit": "GB/s",
                     "frac": algo / (ms * 1e-3) / 1e9 / peak, "traffic": None, "kernel": "normals_knn_kernel",
                     "peak_source": src, "note": "28 B/point algorithmic; the kernel is bound by the k-best search "
                     "(instruction issue), not by HBM"},
        "cpu_baseline": {"value": sample / cpu_s, "unit": "points/s", "cores": oracle.num_threads(),
                         "kind": "reference" if knn.kind == "reference" else "port",
                         "sample": f"kNN (reference nanoflann, OpenMP) + covariance + eigen on {sample} points; "
                                   "kd-tree build not included"},
    }
    return line


def downsample(args, n=10_000_000, bin_size=0.01, ctx=None):
    """PointCloud3f::gridDownsample(bin) on uniform points in the unit cube (~ n * bin^3 ... points per bin)."""
    import oracle
    from cilantro_b200 import synth
    from bench import load_peaks

    capi, ctx = _ctx(ctx)
    pts, _ = synth.kmeans_data(n, 1, seed=3)
    cloud = capi.Cloud(ctx, pts)
    for _ in range(max(args.warmup, 1)):
        cloud.grid_downsample(bin_size).close()
    l0 = ctx.kernel_launches()
    ms_list = []
    m = 0
    for _ in range(args.steps):
        ctx.flush_l2()
        ds = cloud.grid_downsample(bin_size)
        ms_list.append(ds.gpu_ms)
        m = ds.n
        ds.close()
    launches = ctx.kernel_launches() - l0
    ms = float(np.mean(ms_list))
    e2e = []
    for _ in range(3):
        t0 = time.perf_counter()
        capi.grid_downsample(ctx, pts, bin_size)
        e2e.append(time.perf_counter() - t0)
    e2e_s = min(e2e)
    peak, src = load_peaks()
    sample = min(n, 4_000_000)
    t0 = time.perf_counter()
    oracle.grid_downsample(pts[:sample], bin_size, order=2)
    cpu_s = time.perf_counter() - t0
    algo = 12.0 * n + 12.0 * m
    line = {
        "metric": "grid_downsample_points_per_sec", "value": n * 1e3 / ms, "unit": "points/s", "n_gpus": 1,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32 sums, u64 bin keys", "data": "synthetic",
        "config": {"workload": f"PointCloud3f::gridDownsample({bin_size}) on {n} uniform points -> {m} bins",
                   "l2": "flushed before every timed call"},
        "e2e": {"value": n / e2e_s, "unit": "points/s", "h2d_bytes_per_step": pts.nbytes, "d2h_bytes_per_step": 12 * m,
                "what": f"cb_grid_downsample on host arrays (upload + sort + reduce + download): {e2e_s * 1e3:.1f} ms"},
        "gpu_launches": int(launches),
        "roofline": {"bound": "hbm", "achieved": algo / (ms * 1e-3) / 1e9, "peak": peak, "unit": "GB/s",
                     "frac": algo / (ms * 1e-3) / 1e9 / peak, "traffic": None, "kernel": "radix_scatter_kernel (x passes)",
                     "peak_source": src, "note": "algorithmic = 12 B/point read + 12 B/bin written; the sort-based "
                     "implementation moves 12 B (key, index) per point per radix pass on top"},
        "cpu_baseline": {"value": sample / cpu_s, "unit": "points/s", "cores": oracle.num_threads(), "kind": "port",
                         "sample": f"the reference's default parallel std::map build (restated, OpenMP) on {sample} points"},
    }
    return line


def _radius_count_ms(capi, ctx, cloud, r2, reps=5):
    """One cb_radius_search sizing call (one count pass of radius_kernel + a 4 B/point copy of the counts), host clock
    around the synchronising call; median of reps."""
    import ctypes as C

    offsets = np.zeros(cloud.n + 1, np.uint64)
    total = C.c_size_t()
    out = []
    for _ in range(reps + 1):
        ctx.flush_l2()
        ctx.synchronize()
        t0 = time.perf_counter()
        capi._check(capi.lib().cb_radius_search(ctx.h, cloud.h, cloud.h, None, C.c_float(r2), capi._p(offsets), None, None,
                                                C.c_size_t(0), C.byref(total)))
        out.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(out[1:])), int(total.value)


def segment(args, n=1_000_000, k=0, ctx=None):
    """ConnectedComponentExtraction3f::segment on synth.segment_scene, all seeds, normals estimated on the device.
    k == 0: the reference example's recipe (examples/connected_component_extraction.cpp:14-30: radius 0.02 after a
    0.005 downsample = 4 point spacings, NormalsProximityEvaluator 2 degrees, min segment 100) at this scene's spacing;
    k > 0: kNN(k) with AlwaysTrueEvaluator."""
    import oracle
    from oracle import segment as oseg
    from cilantro_b200 import synth
    from bench import load_peaks

    capi, ctx = _ctx(ctx)
    sc = synth.segment_scene(n, seed=1)
    pts, h = sc["points"], sc["spacing"]
    n = pts.shape[0]
    cloud = capi.Cloud(ctx, pts)
    cloud.estimate_normals(k=10, fetch=False)
    r2 = float(np.float32((4.0 * h) ** 2))
    if k == 0:
        kw = dict(radius2=r2, terms=capi.SEG_NORMALS, max_angle=float(np.float32(2.0 * np.pi / 180.0)), min_size=100)
        what = (f"radius {4.0 * h:.5f} (4 spacings), NormalsProximityEvaluator(device normals from kNN(10), 2 deg), "
                f"min segment 100")
    else:
        kw = dict(k=k)
        what = f"kNN({k}), AlwaysTrueEvaluator"
    for _ in range(max(args.warmup, 1)):
        cloud.segment(**kw)
    l0 = ctx.kernel_launches()
    ms_list = []
    for _ in range(args.steps):
        ctx.flush_l2()
        r = cloud.segment(**kw)
        ms_list.append(r["gpu_ms"])
    launches = (ctx.kernel_launches() - l0) // max(args.steps, 1)
    ms = float(np.mean(ms_list))
    # yardstick of "one neighbourhood sweep": only meaningful for the radius row (same cloud, same radius)
    sweep = None
    if k == 0:
        sweep_ms, pairs = _radius_count_ms(capi, ctx, cloud, r2)
        sweep = {"radius_count_ms": sweep_ms, "radius2": r2, "pairs": pairs, "segment_over_count_sweep": ms / sweep_ms,
                 "what": "one cb_radius_search sizing call on the same cloud and radius (radius_kernel count pass + "
                         "4 B/point copy), host clock around the synchronising call"}
    e2e = []
    for _ in range(3):
        t0 = time.perf_counter()
        c2 = capi.Cloud(ctx, pts)
        c2.estimate_normals(k=10, fetch=False)
        c2.segment(**kw)
        e2e.append(time.perf_counter() - t0)
        c2.close()
    e2e_s = min(e2e)
    # CPU baseline and parity: the oracle (serial extractConnectedComponents) on the same input, neighbourhoods from
    # the reference nanoflann (OpenMP). Timed: ONE batched query pass of the reference (kNNSearch, or radiusSearch into
    # rows sized by an untimed count pass) and the extraction. Not timed: the kd-tree build, the count pass and the
    # harness re-sort of the rows on (d2, index).
    nrm = cloud.download(normals=True)[1]
    knn = oracle.make_knn(pts)
    if k > 0:
        t0 = time.perf_counter()
        idx, d2, cnt = knn.neighborhoods(pts, k, oracle.FLT_MAX)
        t_nb = time.perf_counter() - t0
    else:
        _, _, cnt = knn.neighborhoods(pts, 0, r2, stride=1)
        stride = max(1, int(cnt.max()))
        t0 = time.perf_counter()
        idx, d2, cnt = knn.neighborhoods(pts, 0, r2, stride=stride)
        t_nb = time.perf_counter() - t0
    if knn.kind != "port":
        idx, d2 = oseg.sort_rows(idx, d2, cnt)
    ev = {key: kw[key] for key in ("terms", "max_angle", "min_size") if key in kw}
    t0 = time.perf_counter()
    want = oseg.connected_components(pts, nbhd=(idx, d2, cnt), normals=nrm, **ev)
    t_cc = time.perf_counter() - t0
    parity = bool(want["num_clusters"] == r["num_clusters"] and np.array_equal(want["offsets"], r["offsets"]) and
                  np.array_equal(want["points"], r["points"]) and
                  np.array_equal(want["point_to_cluster"], r["point_to_cluster"]))
    peak, src = load_peaks()
    algo = 16.0 * n + 12.0 * n + 4.0 * n  # read the cell-sorted float4 point + float4 normal once, write the labels
    line = {
        "metric": "segmentation_points_per_sec", "value": n * 1e3 / ms, "unit": "points/s", "n_gpus": 1,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32 geometry, u32 union-find", "data": "synthetic",
        "config": {"workload": f"ConnectedComponentExtraction3f::segment on synth.segment_scene({n}): {what}, all seeds "
                               f"-> {r['num_clusters']} segments",
                   "l2": "flushed before every timed call"},
        "e2e": {"value": n / e2e_s, "unit": "points/s", "h2d_bytes_per_step": pts.nbytes, "d2h_bytes_per_step": 16 * n,
                "what": f"cb_cloud_create + cb_cloud_estimate_normals + cb_cloud_segment + labels / CSR on host: "
                        f"{e2e_s * 1e3:.1f} ms"},
        "gpu_launches": int(launches),
        "sweep_yardstick": sweep,
        "roofline": {"bound": "hbm", "achieved": algo / (ms * 1e-3) / 1e9, "peak": peak, "unit": "GB/s",
                     "frac": algo / (ms * 1e-3) / 1e9 / peak, "traffic": None, "kernel": "segment_kernel",
                     "peak_source": src, "note": "32 B/point algorithmic; the sweep is bound by the neighbour search "
                     "(instruction issue and L1 hits on the neighbouring cells), not by HBM; the time includes the "
                     "size filter, two radix sorts and one host read of the segment count"},
        "cpu_baseline": {"value": n / (t_nb + t_cc), "unit": "points/s", "cores": oracle.num_threads(),
                         "kind": "reference" if knn.kind == "reference" else "port",
                         "sample": f"all {n} points: one batched reference query pass {t_nb:.2f} s ("
                                   f"{knn.kind} kd-tree, OpenMP; tree build, row sizing and the (d2, index) re-sort not "
                                   f"included) + serial extraction {t_cc:.2f} s"},
        "parity": {"identical_to_oracle": parity, "points": n, "segments": int(r["num_clusters"])},
    }
    return line


# SASS of plane_score_kernel's plane loop (cuobjdump -sass; two planes per trip of 8 points per thread): 48 FMUL,
# 48 FADD, 16 FSETP, 16 SEL, 8 IADD3 and 18 shared-memory, vote and loop instructions = 154 per 16 point-hypotheses
PLANE_INSTR_PER_POINT_HYP = 154 / 16


def _gpu_facts():
    """Name, power limit and maximum SM clock of GPU 0, read with nvidia-smi (queries only)."""
    import subprocess

    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().split(", ")
    return {"name": q[0], "power_limit_w": float(q[1]), "max_sm_clock_mhz": float(q[2])}


def ransac_plane(args, n=5_000_000, batch=1000, ctx=None):
    """PlaneRANSACEstimator3f on a 5 M-point synth.plane_scene: the step is one batch of 1000 hypotheses through
    cb_plane_score; also a full cb_ransac_plane with an unreachable target (phase split), the reference example's
    recipe end to end, the FP32 issue share, the serial CPU computeResiduals + scan and parity with the oracle."""
    import oracle
    from cilantro_b200 import synth
    from oracle import ransac_plane as orp

    capi, ctx = _ctx(ctx)
    gpu = _gpu_facts()
    sc = synth.plane_scene(n, seed=1)
    pts = sc["points"]
    cloud = capi.Cloud(ctx, pts)
    _, planes = orp.hypotheses(pts, 7, batch)  # the loop's own hypotheses (sample -> closed-form fit)
    for _ in range(max(args.warmup, 1)):
        capi.plane_score(ctx, cloud, planes, 0.01)
    l0 = ctx.kernel_launches()
    times = []
    for _ in range(args.steps):
        ctx.synchronize()
        t0 = time.perf_counter()
        counts = capi.plane_score(ctx, cloud, planes, 0.01)
        times.append(time.perf_counter() - t0)
    launches = ctx.kernel_launches() - l0
    ms = 1e3 * float(np.median(times))
    sms = ctx.device_info()["sm_count"]
    issue_peak = sms * 4 * 32 * gpu["max_sm_clock_mhz"] * 1e6  # thread-instructions per second (4 schedulers per SM)
    instr = PLANE_INSTR_PER_POINT_HYP * n * batch
    # full loop, early exit disabled, and the reference example's recipe (examples/ransac_plane_estimator.cpp)
    full = capi.ransac_plane(ctx, cloud, 11, max_iter=1000, thresh=0.01, inlier_count_thresh=n + 1)
    recipe_kw = dict(max_iter=250, thresh=0.01, inlier_count_thresh=int(0.15 * n))
    capi.ransac_plane(ctx, cloud, 3, **recipe_kw)
    t0 = time.perf_counter()
    recipe = capi.ransac_plane(ctx, cloud, 3, **recipe_kw)
    recipe_s = time.perf_counter() - t0
    # CPU arm: the reference's serial computeResiduals + inlier scan, one hypothesis at a time
    hyp_cpu = 4
    t0 = time.perf_counter()
    oc = [orp.residuals(pts, planes[h], 0.01)[1].size for h in range(hyp_cpu)]
    cpu_s = (time.perf_counter() - t0) / hyp_cpu
    want = orp.ransac_plane(pts, 3, accum_double=True, **recipe_kw)
    parity = {"counts_equal": bool(np.array_equal(oc, counts[:hyp_cpu])), "hypotheses_compared": hyp_cpu,
              "recipe_iterations_equal": recipe["iterations"] == want["iterations"],
              "recipe_best_iteration_equal": recipe["best_iteration"] == want["best_iteration"],
              "recipe_hyp_plane_bits_equal": bool(np.array_equal(recipe["hyp_plane"].view(np.uint32),
                                                                 want["hyp_plane"].view(np.uint32)))}
    parity["all"] = all(v for k, v in parity.items() if k != "hypotheses_compared")
    return {
        "metric": "plane_ransac_hypotheses_per_sec", "value": batch * 1e3 / ms, "unit": "hypotheses/s", "n_gpus": 1,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic", "gpu": gpu,
        "config": {"workload": f"PlaneRANSACEstimator3f scoring: synth.plane_scene({n}) (floor 45 %, wall 25 %, clutter 30 %), "
                               f"{batch} hypotheses per step, thresh 0.01",
                   "l2": "inputs (60 MB) larger than L2; the points are read once per batch"},
        "full_loop": {"iterations": full["iterations"], "ms": full["gpu_ms_total"], "ms_fit": full["gpu_ms_fit"],
                      "ms_score": full["gpu_ms_score"], "ms_reestimate": full["gpu_ms_reestimate"],
                      "ms_final": full["gpu_ms_final"], "num_inliers": full["num_inliers"],
                      "what": "cb_ransac_plane, target n + 1 (no early exit), re-estimation on; device time per phase"},
        "e2e": {"value": recipe["iterations"] / recipe_s, "unit": "hypotheses/s",
                "what": f"the reference example's recipe (thresh 0.01, target 15 %, 250 iterations, re-estimation): "
                        f"{recipe['iterations']} iterations, {recipe['num_inliers']} inliers, {1e3 * recipe_s:.2f} ms host "
                        f"wall clock, {recipe['gpu_ms_total']:.2f} ms device"},
        "gpu_launches": int(launches),
        "roofline": {"bound": "fp32 issue", "achieved": instr / (ms * 1e-3), "peak": issue_peak, "unit": "thread-instr/s",
                     "frac": instr / (ms * 1e-3) / issue_peak, "traffic": None, "kernel": "plane_score_kernel",
                     "peak_source": f"{sms} SMs x 4 warp-instructions x 32 lanes per clock at {gpu['max_sm_clock_mhz']:.0f} MHz",
                     "note": f"{PLANE_INSTR_PER_POINT_HYP:.2f} instructions per point-hypothesis counted in the SASS; "
                             "wall-clock per call incl. 16 KB H2D + 4 KB D2H"},
        "cpu_baseline": {"value": 1.0 / cpu_s, "unit": "hypotheses/s", "cores": 1, "kind": "port",
                         "sample": f"serial computeResiduals + scan over all {n} points, {hyp_cpu} hypotheses "
                                   f"({1e3 * cpu_s:.1f} ms each; {batch} would take {batch * cpu_s:.1f} s)"},
        "parity": parity,
    }


def _pca_parity(g, o, sample):
    def get(d, *names):
        for nm in names:
            if nm in d:
                return np.asarray(d[nm], np.float64)
        return None

    out = {"points": int(sample),
           "note": "the CPU arm sums 10^7 fp32 terms serially in fp32 like the reference (covariance.hpp:64-76); the device "
                   "accumulates in double, so the differences are the CPU arm's rounding"}
    gm, om = get(g, "mean"), get(o, "mean")
    gc, oc = get(g, "cov", "covariance"), get(o, "cov", "covariance")
    ge, oe = get(g, "eigenvalues", "evals"), get(o, "eigenvalues", "evals")
    if gm is not None and om is not None:
        out["mean_max_abs_diff"] = float(np.abs(gm.ravel() - om.ravel()).max())
    if gc is not None and oc is not None:
        out["cov_max_abs_diff"] = float(np.abs(gc.ravel() - oc.ravel()).max())
    if ge is not None and oe is not None:
        out["eigenvalue_max_abs_diff"] = float(np.abs(ge.ravel() - oe.ravel()).max())
    return out


def meanshift(args, blobs=1000, per_blob=1000, ctx=None):
    """MeanShift3f::cluster on synth.mean_shift_scene(blobs, per_blob, sigma=1), every point a seed, the reference
    example's recipe (kernel radius 2 sigma, cluster tol 0.2 sigma, flat kernel), max_iter 100. One step = one call."""
    import oracle
    from oracle import mean_shift as oms
    from cilantro_b200 import synth

    capi, ctx = _ctx(ctx)
    sc = synth.mean_shift_scene(blobs, per_blob, sigma=1.0, seed=1)
    pts = sc["points"]
    n = pts.shape[0]
    radius, max_iter, ctol = 2.0, 100, 0.2
    cloud = capi.Cloud(ctx, pts)
    for _ in range(max(args.warmup, 1)):
        cloud.mean_shift(radius, max_iter, ctol)
    l0 = ctx.kernel_launches()
    ms_list, shift_list = [], []
    for _ in range(args.steps):
        ctx.flush_l2()
        r = cloud.mean_shift(radius, max_iter, ctol)
        ms_list.append(r["gpu_ms"])
        shift_list.append(r["gpu_ms_shift"])
    launches = (ctx.kernel_launches() - l0) // max(args.steps, 1)
    ms, ms_shift = float(np.mean(ms_list)), float(np.mean(shift_list))
    r2 = float(np.float32(radius) * np.float32(radius))
    count_ms, pairs = _radius_count_ms(capi, ctx, cloud, r2)
    # device time per kernel of one call (torch.profiler, CUDA activities, in a run of its own)
    kernels = None
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            cloud.mean_shift(radius, max_iter, ctol)
            torch.cuda.synchronize()
        acc = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                name = e.name.replace("(anonymous namespace)::", "").replace("void ", "").split("(")[0]
                acc[name] = acc.get(name, 0.0) + e.device_time_total / 1e3
        kernels = {k: round(v, 3) for k, v in sorted(acc.items(), key=lambda kv: -kv[1])[:12]}
    except Exception as exc:  # the profiler is diagnostic only: the timed numbers above do not depend on it
        kernels = {"error": repr(exc)}
    # CPU arm: one reference nanoflann radius pass (OpenMP) over a seeded 1 % sample of the seeds at the first
    # iteration's positions; the seeds are independent, so this is the per-seed rate of one full shift iteration.
    rng = np.random.default_rng(7)
    sample = np.sort(rng.choice(n, n // 100, replace=False))
    knn = oracle.make_knn(pts)
    _, _, cnt = knn.neighborhoods(pts[sample], 0, r2, stride=1)
    stride = max(1, int(cnt.max()))
    t0 = time.perf_counter()
    knn.neighborhoods(pts[sample], 0, r2, stride=stride)
    t_sample = time.perf_counter() - t0
    cpu_iter_ms = t_sample * 1e3 * n / sample.size
    # parity inside the run: the oracle's shift of 200 sampled seeds (bit for bit) and the oracle's clustering of the
    # device's shifted seeds (labels, CSR and modes)
    few = np.sort(rng.choice(n, 200, replace=False))
    want = oms.mean_shift(pts, radius, r["iterations"], ctol, seeds=pts[few])
    shift_ok = bool(np.array_equal(want["shifted_seeds"].view(np.uint32), r["shifted_seeds"][few].view(np.uint32)))
    wc = oms.mean_shift(pts, radius, 0, ctol, seeds=r["shifted_seeds"])
    cluster_ok = bool(all(np.array_equal(wc[k], r[k]) for k in ("offsets", "points", "point_to_cluster")) and
                      np.array_equal(wc["modes"].view(np.uint32), r["modes"].view(np.uint32)))
    return {
        "metric": "meanshift_ms_per_call", "value": ms, "unit": "ms", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": False, "dtype": "f32", "data": "synthetic",
        "config": {"workload": f"MeanShift3f::cluster on synth.mean_shift_scene({blobs}, {per_blob}, sigma 1): {n} seeds, "
                               f"kernel radius {radius}, cluster tol {ctol}, flat kernel, max_iter {max_iter}",
                   "l2": "flushed before every timed call"},
        "iterations": r["iterations"], "clusters": r["num_clusters"], "gpu_launches": int(launches),
        "ms_shift": ms_shift, "ms_cluster": ms - ms_shift, "ms_per_iteration": ms_shift / max(r["iterations"], 1),
        "kernel_ms_one_call": kernels,
        "sweep_yardstick": {"radius_count_ms": count_ms, "pairs": pairs,
                            "what": "one cb_radius_search sizing call on the same cloud at the kernel radius"},
        "cpu_baseline": {"ms_per_full_iteration": cpu_iter_ms, "sample_seeds": int(sample.size), "sample_s": t_sample,
                         "impl": knn.kind, "threads": oracle.num_threads(),
                         "what": "reference nanoflann radiusSearch over a 1 % seed sample at the starting positions, "
                                 "scaled to all seeds (one shift iteration; the weighted sums are not timed)"},
        "parity": {"sampled_shifted_seeds_bit_exact": shift_ok, "oracle_clustering_of_gpu_seeds_identical": cluster_ok},
    }


AUX = {"downsample_10m": downsample, "downsample_1m": lambda a: downsample(a, n=1_000_000, bin_size=0.02),
       "normals_5m": normals, "normals_1m": lambda a: normals(a, n=1_000_000),
       "kmeans_50m": kmeans, "ransac_5m": ransac, "pca_50m": pca,
       "kmeans_5m": lambda a: kmeans(a, n=5_000_000, k=256), "ransac_500k": lambda a: ransac(a, n=500_000, batch=256),
       "pca_5m": lambda a: pca(a, n=5_000_000),
       "segment_1m": segment, "segment_knn_1m": lambda a: segment(a, k=10), "meanshift_1m": meanshift,
       "ransac_plane_5m": ransac_plane}
