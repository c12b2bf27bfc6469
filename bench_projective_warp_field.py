"""Projective correspondence search of the warp-field ICPs (cb_warp_icp_set_projection,
cb_sparse_warp_icp_set_projection, DESIGN §4.22) against their grid search on the same frame pair: per ICP iteration
the search, the Gauss-Newton step (assembly and CG; the dense object reports them together with compose as `solve`),
the sparse resampling, and the launches; per attach the index map's build time.

    python bench_projective_warp_field.py [--iters 5] [--repeats 3]

Workloads: a bending sheet 1 m in front of the camera, rendered at 640 x 480 and at 1920 x 1080 from a dense sampling,
converted back with normals on the device; the first frame is the destination, the third (bent by another 8 mm at
the edges) the source. The sparse recipe (2.5 cm control nodes, 4-NN control lists, 8-NN node neighbourhoods) and the
dense recipe (12-NN neighbourhoods) of the reference's examples/non_rigid_icp.cpp run a fixed number of iterations
(tol = 0). Times are CUDA-event times reported by the objects, medians over repeats, per iteration; `build_ms` is the
median host time of the attach, which ends with a stream synchronise. Prints one JSON line with the card's name and
power limit; writes nothing."""
import argparse
import json
import subprocess
import time

import numpy as np

from cilantro_b200 import capi

F = np.float32
SIZES = [(640, 480), (1920, 1080)]
SPARSE = dict(w_pt=0.0, w_pl=1.0, stiffness=200.0, huber=1e-2, max_gn_iter=1, gn_tol=5e-4, max_cg_iter=500,
              cg_tol=1e-5, reg_sigma=0.075, ctrl_sigma=0.0125, max_d2=F(0.02 * 0.02), tol=0.0)
DENSE = dict(w_pt=0.1, w_pl=1.0, stiffness=200.0, huber=1e-2, max_gn_iter=1, gn_tol=5e-4, max_cg_iter=500, cg_tol=1e-5,
             reg_sigma=0.015, max_d2=F(0.04 * 0.04), tol=0.0)


def gpu_info():
    """(name, power limit W) of GPU 0, read with nvidia-smi."""
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=60, check=True).stdout
    name, power = [x.strip() for x in out.strip().splitlines()[0].split(",")]
    return name, float(power)


def sheet(k, n):
    x, y = np.meshgrid(np.linspace(-0.4, 0.4, n), np.linspace(-0.3, 0.3, n))
    z = 1.0 + 0.02 * np.sin(6 * x) * np.cos(5 * y) + 0.004 * k * (x / 0.4) ** 2 - 0.002 * k * (y / 0.3)
    return np.stack([x, y, z], -1).reshape(-1, 3).astype(F)


def timed(obj, kw, repeats, keys):
    obj.estimate(**kw)  # warm-up
    rows = []
    for _ in range(repeats):
        r = obj.estimate(**kw)
        it = r["iterations"]
        rows.append({k: r[k] / it for k in keys} | {"launches": r["kernel_launches"] / it, "num_corr": r["num_corr"]})
    return {k: float(np.median([r[k] for r in rows])) for k in rows[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    name, power = gpu_info()
    ctx = capi.Context(0)
    conv = capi.DepthConverter(np.float32, 1.0)
    out = []
    for w, h in SIZES:
        f = 0.82 * w * 1.0 / 0.8
        K = np.array([[f, 0, (w - 1) / 2], [0, f, (h - 1) / 2], [0, 0, 1]], F)
        n = int(1.6 * w)
        frames = []
        for k in (0, 2):
            depth = capi.points_to_depth_image(ctx, sheet(k, n), K, w, h, conv)
            r = capi.depth_image_to_points(ctx, depth, K, conv, normals=True)
            frames.append((r["points"], r["normals"]))
        dst = capi.Cloud(ctx, *frames[0])
        src = capi.Cloud(ctx, frames[1][0])
        nodes = src.grid_downsample(0.025)
        ctrl = capi.neighborhood_csr(*capi.knn_radius(ctx, nodes, src, 4))
        reg = capi.neighborhood_csr(*capi.knn_radius(ctx, nodes, nodes, 8))
        nb = capi.neighborhood_csr(*capi.knn_radius(ctx, src, src, 12))
        row = dict(frame=f"{w}x{h}", dst_points=int(dst.n), src_points=int(src.n), nodes=int(nodes.n))
        for label, make, kw, keys in (
                ("sparse", lambda: capi.SparseWarpIcp(ctx, dst, src, ctrl, nodes.n, reg), SPARSE,
                 ("gpu_ms_search", "gpu_ms_assemble", "gpu_ms_cg", "gpu_ms_resample")),
                ("dense", lambda: capi.WarpIcp(ctx, dst, src, *nb), DENSE, ("gpu_ms_search", "gpu_ms_solve"))):
            kw = dict(kw, max_iter=args.iters)
            proj, grid = make(), make()
            build = []
            for _ in range(args.repeats + 1):
                t0 = time.perf_counter()
                proj.set_projection(K, w, h)
                build.append((time.perf_counter() - t0) * 1e3)
            row[label] = dict(build_ms=float(np.median(build[1:])), projective=timed(proj, kw, args.repeats, keys),
                              grid=timed(grid, kw, args.repeats, keys))
            proj.close()
            grid.close()
        out.append(row)
    ctx.close()
    print(json.dumps({"gpu": name, "power_limit_w": power, "iters": args.iters, "results": out}))


if __name__ == "__main__":
    main()
