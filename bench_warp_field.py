"""Dense rigid warp-field ICP (SimpleCombinedMetricDenseRigidWarpFieldICP3f) on one GPU: one JSON line in the shape
of the bench_aux workloads.

    python bench_warp_field.py --workload warp_icp_100k [--steps 3 --warmup 1]
    python bench_warp_field.py --workload warp_icp_1m

Workload: synth.warp_pair(n) at a 5 mm mean spacing (warp_icp_100k: roughly a scan downsampled at 5 mm), 12-NN
regularisation neighbourhoods over the source (cb_knn_radius), and the dense recipe of the reference example
(examples/non_rigid_icp.cpp): sigma 3 res, w_pt 0.1, w_pl 1, stiffness 200, Huber 1e-2, max distance 0.04, 15
iterations, tolerance 2.5e-3, 1 Gauss-Newton step, 500 CG iterations. L2 is flushed before each timed call. The CPU
arm is the oracle's serial fp32 restatement (the reference needs Eigen), timed for one ICP iteration on at most 100 k
points and not scaled. Writes nothing to the tree.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

RES = 0.005
RECIPE = dict(w_pt=0.1, w_pl=1.0, stiffness=200.0, huber=1e-2, reg_sigma=3 * RES, max_iter=15, tol=2.5e-3,
              max_d2=0.04 ** 2, max_gn_iter=1, gn_tol=5e-4, max_cg_iter=500, cg_tol=1e-5)
WORKLOADS = {"warp_icp_100k": 100_000, "warp_icp_1m": 1_000_000}
HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s


def cg_bytes_per_iteration(n, incidences):
    """Bytes one CG iteration moves, from the shapes (fp32 vectors of 6 per point; one matvec reads B_i (21 floats),
    p_i, the incidence range and per incidence the arc id, the other end, c_e (6) and the other end's p (6), and
    writes q_i; the update reads x, r, p, q and the preconditioner and writes x, r, z; the direction update reads z, p
    and writes p)."""
    matvec = n * (21 * 4 + 24 + 4 + 24) + incidences * (4 + 4 + 24 + 24)
    update = n * 24 * (5 + 3)
    direction = n * 24 * 3
    return matvec + update + direction


def neighbourhoods(capi, ctx, cloud, k=12):
    idx, d2, cnt = capi.knn_radius(ctx, cloud, cloud, k)
    return capi.neighborhood_csr(idx, d2, cnt)


def run(args):
    from bench_aux import _gpu_facts
    from cilantro_b200 import capi, synth

    n = WORKLOADS[args.workload]
    ctx = capi.Context(0)
    gpu = _gpu_facts()
    P = synth.warp_pair(n, seed=1, spacing=RES)
    dst = capi.Cloud(ctx, P["dst"], P["dst_normals"])
    src = capi.Cloud(ctx, P["src"])
    nb = neighbourhoods(capi, ctx, src)
    icp = capi.WarpIcp(ctx, dst, src, *nb)
    incidences = 2 * int(np.count_nonzero(nb[1] != np.repeat(nb[1][nb[0][:-1].astype(np.int64)],
                                                              np.diff(nb[0].astype(np.int64)))))
    for _ in range(max(args.warmup, 1)):
        icp.estimate(**RECIPE)
    times, res = [], None
    for _ in range(args.steps):
        ctx.flush_l2()
        ctx.synchronize()
        t0 = time.perf_counter()
        res = icp.estimate(**RECIPE)
        times.append(time.perf_counter() - t0)
    ms = 1e3 * float(np.median(times))
    # ms per CG iteration: one Gauss-Newton step with 500 and with 0 CG iterations (cg_tol 0), same correspondences
    f, s, _ = icp.correspondences()
    kw_cg = dict(RECIPE, cg_tol=0.0)
    icp.solve(f, s, **dict(kw_cg, max_cg_iter=500))
    walls = {}
    for m in (0, 500):
        w = []
        for _ in range(3):
            ctx.flush_l2()
            ctx.synchronize()
            t0 = time.perf_counter()
            icp.solve(f, s, **dict(kw_cg, max_cg_iter=m))
            w.append(time.perf_counter() - t0)
        walls[m] = float(np.median(w))
    cg_ms = 1e3 * (walls[500] - walls[0]) / 500
    cg_bytes = cg_bytes_per_iteration(n, incidences)
    # kernel time of one call, torch.profiler in a run of its own
    kernel_ms = None
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile

        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            icp.estimate(**RECIPE)
            ctx.synchronize()
        kernel_ms = sum(e.device_time_total for e in prof.key_averages()) / 1e3
    except Exception as e:  # noqa: BLE001 (reported, not hidden)
        kernel_ms = f"not measured: {type(e).__name__}: {e}"
    # CPU arm: the oracle's serial fp32 estimator for one ICP iteration (search excluded), on at most 100 k points
    import oracle
    from oracle import warp_field as owf

    m = min(n, 100_000)
    okw = {k: v for k, v in RECIPE.items() if k not in ("max_iter", "tol", "max_d2", "huber")}
    okw["huber_delta"] = RECIPE["huber"]
    Pm = P if m == n else synth.warp_pair(m, seed=1, spacing=RES)
    if m == n:
        sel_f, sel_s, nbm = *icp.correspondences()[:2], nb
    else:
        src_m = capi.Cloud(ctx, Pm["src"])
        nbm = neighbourhoods(capi, ctx, src_m)
        sel_f, sel_s, _ = capi.find_correspondences(ctx, dst if m == n else capi.Cloud(ctx, Pm["dst"]), src_m, None,
                                                    RECIPE["max_d2"])
    ic = capi.WarpIcp(ctx, capi.Cloud(ctx, Pm["dst"], Pm["dst_normals"]), capi.Cloud(ctx, Pm["src"]), *nbm)
    t0 = time.perf_counter()
    o = owf.solve(Pm["dst"], Pm["dst_normals"], Pm["src"], sel_f, sel_s, nbm, **okw)
    cpu_s = time.perf_counter() - t0
    g = ic.solve(sel_f, sel_s, **{k: v for k, v in RECIPE.items() if k not in ("max_iter", "tol", "max_d2")})
    # parity of the whole loop against the oracle on a seeded subsample
    Ps = synth.warp_pair(1500, seed=11, spacing=RES)
    idx, d2, cnt = oracle.BruteKnn(Ps["src"]).neighborhoods(Ps["src"], 12, 3.0e38)
    nbs = capi.neighborhood_csr(idx, d2, cnt)
    gs = capi.WarpIcp(ctx, capi.Cloud(ctx, Ps["dst"], Ps["dst_normals"]), capi.Cloud(ctx, Ps["src"]), *nbs).estimate(**RECIPE)
    okw_loop = dict(okw, max_iter=RECIPE["max_iter"], tol=RECIPE["tol"], max_d2=RECIPE["max_d2"])
    os_ = owf.icp(Ps["dst"], Ps["dst_normals"], Ps["src"], nbs, **okw_loop)
    warped_err = float(np.abs(owf.apply(gs["T"], Ps["src"]) - owf.apply(os_["T"], Ps["src"])).max())
    parity = {"points": 1500, "iterations_equal": gs["iterations"] == os_["iterations"],
              "max_warped_point_difference_m": warped_err,
              "one_step_max_transform_difference": float(np.abs(g["T"] - o["T"]).max()),
              "one_step_cg_iterations": [g["cg_iterations"], o["cg_iterations"]]}
    parity["all"] = parity["iterations_equal"] and warped_err < 1e-5
    ms_iter = ms / max(res["iterations"], 1)
    line = {
        "metric": "warp_icp_ms_per_call", "value": ms, "unit": "ms", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": False, "dtype": "f32", "data": "synthetic",
        "gpu": gpu,
        "config": {"workload": f"{args.workload}: synth.warp_pair({n}), 5 mm spacing, 12-NN regularisation, the reference "
                               "example's dense recipe", "l2": "flushed before every timed call",
                   "incidences": incidences},
        "iterations": res["iterations"], "num_corr": res["num_corr"], "gn_steps": res["gn_steps"],
        "cg_iterations": res["cg_iterations"],
        "cg_iterations_per_gn_step": res["cg_iterations"] / max(res["gn_steps"], 1),
        "ms_per_icp_iteration": ms_iter, "ms_per_cg_iteration": cg_ms,
        "device_ms": {"search": res["gpu_ms_search"], "solve": res["gpu_ms_solve"]},
        "gpu_launches": res["kernel_launches"], "kernel_ms_one_call": kernel_ms,
        "roofline": {"bound": "HBM bandwidth", "bytes_per_cg_iteration": cg_bytes,
                     "achieved": cg_bytes / (cg_ms * 1e-3) if cg_ms > 0 else None, "peak": HBM_PEAK, "unit": "B/s",
                     "frac": cg_bytes / (cg_ms * 1e-3) / HBM_PEAK if cg_ms > 0 else None,
                     "note": "bytes from the shapes (each operand once per CG iteration); time = wall-clock difference of "
                             "one Gauss-Newton step with 500 and 0 CG iterations, divided by 500"},
        "cpu_baseline": {"value": cpu_s * 1e3, "unit": "ms", "kind": "oracle fp32 restatement, serial (not the reference)",
                         "sample": f"one ICP iteration's estimator (1 Gauss-Newton step, {o['cg_iterations']} CG iterations) "
                                   f"on {m} points, search excluded; not scaled to a full call"},
        "parity": parity,
    }
    ctx.close()
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=sorted(WORKLOADS), default="warp_icp_100k")
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    print(json.dumps(run(args)))


if __name__ == "__main__":
    main()
