"""Sparse rigid warp-field ICP (SimpleCombinedMetricSparseRigidWarpFieldICP3f) on one GPU: one JSON line in the shape
bench_warp_field.py prints.

    python bench_sparse_warp_field.py --workload sparse_warp_icp_120k [--steps 3 --warmup 1]
    python bench_sparse_warp_field.py --workload sparse_warp_icp_1m

Workload: synth.warp_pair(n) at a 5 mm mean spacing with no source downsampling (sparse_warp_icp_120k: the scale of
the reference example's scans), control nodes = the source grid-downsampled at 2.5 cm on the device, 4-NN control
lists and 8-NN node neighbourhoods (cb_knn_radius), and the sparse recipe of the reference example
(examples/non_rigid_icp.cpp:41-82): control sigma 0.5 res, regularisation sigma 3 res, w_pt 0, w_pl 1, stiffness 200,
Huber 1e-2, max distance 0.02, 15 iterations, tolerance 2.5e-3, 1 Gauss-Newton step, 500 CG iterations. L2 is flushed
before each timed call. The CPU arm is the oracle's serial fp32 restatement (not the reference, which needs Eigen),
timed for one ICP iteration's estimator on at most 100 k points and not scaled. Writes nothing to the tree.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

RES = 0.025
RECIPE = dict(w_pt=0.0, w_pl=1.0, stiffness=200.0, huber=1e-2, reg_sigma=3 * RES, ctrl_sigma=0.5 * RES, max_iter=15,
              tol=2.5e-3, max_d2=0.02 ** 2, max_gn_iter=1, gn_tol=5e-4, max_cg_iter=500, cg_tol=1e-5)
WORKLOADS = {"sparse_warp_icp_120k": 120_000, "sparse_warp_icp_1m": 1_000_000}
HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s


def cg_bytes_per_iteration(n, m, entries, incidences):
    """Bytes one CG iteration moves, from the shapes (fp32 vectors of 6 per node). Point half of the matvec: per point
    the list range, per entry its weight, node and the node's p (6), B_i (21) and y_i (6) written. Node half: per node
    the two ranges, per node-incidence the entry, its weight, the point and y_i (6), per arc incidence the arc id, the
    other end, c_e (6) and the other end's p (6), p_j read and q_j written. The update reads x, r, p, q and the
    preconditioner and writes x, r, z; the direction update reads z, p and writes p."""
    point_half = n * (8 + 21 * 4 + 24) + entries * (4 + 4 + 24)
    node_half = m * (16 + 24 + 24) + entries * (4 + 4 + 4 + 24) + incidences * (4 + 4 + 24 + 24)
    return point_half + node_half + m * 24 * 8 + m * 24 * 3


def setup(capi, ctx, n, seed=1):
    from cilantro_b200 import synth

    P = synth.warp_pair(n, seed=seed, spacing=0.005)
    dst = capi.Cloud(ctx, P["dst"], P["dst_normals"])
    src = capi.Cloud(ctx, P["src"])
    nodes = src.grid_downsample(RES)
    ctrl = capi.neighborhood_csr(*capi.knn_radius(ctx, nodes, src, 4))
    reg = capi.neighborhood_csr(*capi.knn_radius(ctx, nodes, nodes, 8))
    return P, dst, src, nodes, ctrl, reg


def arc_incidences(reg):
    off, idx, _ = reg
    centre = np.repeat(idx[off[:-1].astype(np.int64)], np.diff(off.astype(np.int64)))
    return 2 * int(np.count_nonzero(idx != centre))


def run(args):
    from bench_aux import _gpu_facts
    from cilantro_b200 import capi

    n = WORKLOADS[args.workload]
    ctx = capi.Context(0)
    gpu = _gpu_facts()
    P, dst, src, nodes, ctrl, reg = setup(capi, ctx, n)
    m = nodes.n
    icp = capi.SparseWarpIcp(ctx, dst, src, ctrl, m, reg)
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
    Td = res["T_dense"]
    kw_cg = {k: v for k, v in RECIPE.items() if k not in ("max_iter", "tol", "max_d2")}
    kw_cg["cg_tol"] = 0.0
    icp.solve(f, s, T_dense_src=Td, **dict(kw_cg, max_cg_iter=500))
    walls = {}
    for it in (0, 500):
        w = []
        for _ in range(3):
            ctx.flush_l2()
            ctx.synchronize()
            t0 = time.perf_counter()
            icp.solve(f, s, T_dense_src=Td, **dict(kw_cg, max_cg_iter=it))
            w.append(time.perf_counter() - t0)
        walls[it] = float(np.median(w))
    cg_ms = 1e3 * (walls[500] - walls[0]) / 500
    entries, incidences = int(ctrl[0][-1]), arc_incidences(reg)
    cg_bytes = cg_bytes_per_iteration(n, m, entries, incidences)
    # CPU arm: the oracle's serial fp32 estimator for one ICP iteration (search excluded), on at most 100 k points
    from oracle import sparse_warp_field as osw

    okw = {k: v for k, v in RECIPE.items() if k not in ("max_iter", "tol", "max_d2", "huber")}
    okw["huber_delta"] = RECIPE["huber"]
    nc = min(n, 100_000)
    Pc, dc, sc_, nodes_c, ctrl_c, reg_c = setup(capi, ctx, nc)
    fc, scorr, _ = capi.find_correspondences(ctx, dc, sc_, None, RECIPE["max_d2"])
    t0 = time.perf_counter()
    o = osw.solve(Pc["dst"], Pc["dst_normals"], Pc["src"], fc, scorr, ctrl_c, nodes_c.n, reg_c, **okw)
    cpu_s = time.perf_counter() - t0
    g = capi.SparseWarpIcp(ctx, dc, sc_, ctrl_c, nodes_c.n, reg_c).solve(fc, scorr, **{
        k: v for k, v in RECIPE.items() if k not in ("max_iter", "tol", "max_d2")})
    # parity of the whole loop against the oracle on a seeded subsample
    Ps, ds, ss, nodes_s, ctrl_s, reg_s = setup(capi, ctx, 3000, seed=11)
    gs = capi.SparseWarpIcp(ctx, ds, ss, ctrl_s, nodes_s.n, reg_s).estimate(**RECIPE)
    os_ = osw.icp(Ps["dst"], Ps["dst_normals"], Ps["src"], ctrl_s, nodes_s.n, reg_s,
                  **dict(okw, max_iter=RECIPE["max_iter"], tol=RECIPE["tol"], max_d2=RECIPE["max_d2"]))
    warped_err = float(np.abs(osw.apply(gs["T_dense"], Ps["src"]) - osw.apply(os_["T_dense"], Ps["src"])).max())
    parity = {"points": 3000, "nodes": nodes_s.n, "iterations_equal": gs["iterations"] == os_["iterations"],
              "max_warped_point_difference_m": warped_err,
              "one_step_max_transform_difference": float(np.abs(g["T"] - o["T"]).max()),
              "one_step_cg_iterations": [g["cg_iterations"], o["cg_iterations"]]}
    parity["all"] = bool(parity["iterations_equal"] and warped_err < 1e-5 and
                         parity["one_step_max_transform_difference"] < 1e-5)
    ms_iter = ms / max(res["iterations"], 1)
    line = {
        "metric": "sparse_warp_icp_ms_per_call", "value": ms, "unit": "ms", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": False, "dtype": "f32", "data": "synthetic",
        "gpu": gpu,
        "config": {"workload": f"{args.workload}: synth.warp_pair({n}), 5 mm spacing, no source downsampling, "
                               f"{m} control nodes at 2.5 cm, 4-NN control lists, 8-NN node neighbourhoods, the "
                               "reference example's sparse recipe", "l2": "flushed before every timed call",
                   "control_entries": entries, "arc_incidences": incidences},
        "iterations": res["iterations"], "num_corr": res["num_corr"], "gn_steps": res["gn_steps"],
        "cg_iterations": res["cg_iterations"],
        "cg_iterations_per_gn_step": res["cg_iterations"] / max(res["gn_steps"], 1),
        "ms_per_icp_iteration": ms_iter, "ms_per_cg_iteration": cg_ms,
        "device_ms": {"search": res["gpu_ms_search"], "resample": res["gpu_ms_resample"],
                      "assembly": res["gpu_ms_assemble"], "cg": res["gpu_ms_cg"]},
        "gpu_launches": res["kernel_launches"],
        "roofline": {"bound": "HBM bandwidth", "bytes_per_cg_iteration": cg_bytes,
                     "achieved": cg_bytes / (cg_ms * 1e-3) if cg_ms > 0 else None, "peak": HBM_PEAK, "unit": "B/s",
                     "frac": cg_bytes / (cg_ms * 1e-3) / HBM_PEAK if cg_ms > 0 else None,
                     "note": "bytes from the shapes (each operand once per CG iteration); time = wall-clock difference of "
                             "one Gauss-Newton step with 500 and 0 CG iterations, divided by 500"},
        "cpu_baseline": {"value": cpu_s * 1e3, "unit": "ms", "kind": "oracle fp32 restatement, serial (not the reference)",
                         "sample": f"one ICP iteration's estimator (1 Gauss-Newton step, {o['cg_iterations']} CG iterations) "
                                   f"on {nc} points, search excluded; not scaled to a full call"},
        "parity": parity,
    }
    ctx.close()
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=sorted(WORKLOADS), default="sparse_warp_icp_120k")
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    print(json.dumps(run(args)))


if __name__ == "__main__":
    main()
