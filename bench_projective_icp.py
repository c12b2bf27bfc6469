"""Projective rigid ICP on the device (cb_icp_set_projection, DESIGN §4.21) against the kd-tree combined ICP on the same
inputs: device time per iteration, launches per iteration, the index map's build time, and bytes over time.

    python bench_projective_icp.py [--iters 10] [--repeats 5]

Workloads: a synthetic room (floor, ceiling, three walls) sampled at about 1 M and 2 M points with exact normals is the
model (destination); a 640 x 480 and a 1920 x 1080 float depth frame ray-cast against the same planes from a camera
pose off the model's and converted back with normals on the device is the source, as in the fusion example's
localisation step. Both ICPs run the combined metric with the plane term only (SimpleCombinedMetricRigidProjectiveICP3f's weights),
max_d2 = 0.1^2, a fixed number of iterations (tol = 0), on the device-resident loop. `iter_ms` is the median over
repeats of the CUDA-event-bracketed iterations' mean; `build_ms` is the median host time of cb_icp_set_projection, which
ends with a stream synchronise. Bytes per projective iteration are the minimum the pass reads: per source point its
packed coordinates (12 B) and one map entry (4 B), per matched point the destination point and normal (24 B); they are
set against NVIDIA's H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s (a data-sheet figure, not a measurement).
Prints one JSON line; writes nothing."""
import argparse
import json
import subprocess
import time

import numpy as np

from cilantro_b200 import capi

HBM_BPS = 3.35e12
F = np.float32
WORKLOADS = [((640, 480), 1.0e6), ((1920, 1080), 2.0e6)]


def gpu_info():
    """(name, power limit W) of GPU 0, read with nvidia-smi."""
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=60, check=True).stdout
    name, power = [x.strip() for x in out.strip().splitlines()[0].split(",")]
    return name, float(power)


def room(n_target):
    """About n_target points on a 4 x 2.4 x 5 m room's floor, ceiling and three walls, with their normals."""
    planes = [([-2, 1.2, 0], [1, 0, 0], [0, 0, 1], 4.0, 5.0, [0, -1, 0]),
              ([-2, -1.2, 0], [1, 0, 0], [0, 0, 1], 4.0, 5.0, [0, 1, 0]),
              ([-2, -1.2, 5], [1, 0, 0], [0, 1, 0], 4.0, 2.4, [0, 0, -1]),
              ([-2, -1.2, 0], [0, 1, 0], [0, 0, 1], 2.4, 5.0, [1, 0, 0]),
              ([2, -1.2, 0], [0, 1, 0], [0, 0, 1], 2.4, 5.0, [-1, 0, 0])]
    s = np.sqrt(sum(a * b for _, _, _, a, b, _ in planes) / n_target)
    pts, nrm = [], []
    for o, u, v, a, b, n in planes:
        x, y = np.meshgrid(np.arange(0, a, s), np.arange(0, b, s))
        p = np.asarray(o) + x.reshape(-1, 1) * np.asarray(u) + y.reshape(-1, 1) * np.asarray(v)
        pts.append(p)
        nrm.append(np.tile(n, (p.shape[0], 1)))
    return np.vstack(pts).astype(F), np.vstack(nrm).astype(F)


def ray_cast(K, w, h, P):
    """The float depth image of the room's planes seen from camera pose P: every pixel hits a wall, so the frame is as
    dense as the image (a rendering of the sampled model would leave most 1920 x 1080 pixels empty)."""
    v, u = np.mgrid[0:h, 0:w].astype(np.float64)
    d = np.stack([u, v, np.ones_like(u)], -1) @ np.linalg.inv(np.asarray(K, np.float64)).T  # camera rays, z = 1
    R, o = np.asarray(P[:, :3], np.float64), np.asarray(P[:, 3], np.float64)
    dw = d @ R.T
    t = np.full((h, w), np.inf)
    for axis, c in ((1, 1.2), (1, -1.2), (2, 5.0), (0, -2.0), (0, 2.0)):
        with np.errstate(divide="ignore", invalid="ignore"):
            tc = (c - o[axis]) / dw[..., axis]
        t = np.where((tc > 0) & (tc < t), tc, t)
    return np.where(np.isfinite(t), t, 0).astype(F)  # camera-frame z = t, since the rays have z = 1


def pose(angle, t):
    ax = np.array([0.3, -0.8, 0.5]) / np.linalg.norm([0.3, -0.8, 0.5])
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    R = np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K
    return np.hstack([R, np.asarray(t, np.float64)[:, None]]).astype(F)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    name, power = gpu_info()
    ctx = capi.Context(0)
    conv = capi.DepthConverter(np.float32, 1.0)
    kw = dict(metric="combined", w_pt=0.0, w_pl=1.0, max_d2=F(0.1 * 0.1), max_iter=args.iters, tol=0.0, timing=1)
    rows = []
    for (w, h), n_model in WORKLOADS:
        f = 0.825 * w
        K = np.array([[f, 0, (w - 1) / 2], [0, f, (h - 1) / 2], [0, 0, 1]], F)
        pts, nrm = room(n_model)
        model = capi.Cloud(ctx, pts, nrm)
        P = pose(0.01, [0.02, -0.01, 0.03])
        depth = ray_cast(K, w, h, P)
        frame = capi.depth_image_to_points(ctx, depth, K, conv, normals=True, to_device=True)["cloud"]
        cam0 = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(F)
        proj = capi.Icp(ctx, model, frame)
        build = []
        for _ in range(args.repeats + 1):
            t0 = time.perf_counter()
            proj.set_projection(K, w, h, cam0)
            build.append((time.perf_counter() - t0) * 1e3)
        kd = capi.Icp(ctx, model, frame)
        res = {}
        for label, icp in (("projective", proj), ("kdtree", kd)):
            icp.estimate(**kw)  # warm-up: packed copies, module load
            ms, launches, corr = [], 0, 0
            for _ in range(args.repeats):
                r = icp.estimate(**kw)
                ms.append(r["gpu_ms_total"] / r["iterations"])
                launches, corr = r["kernel_launches"] / r["iterations"], r["num_corr"]
            res[label] = dict(iter_ms=float(np.median(ms)), launches_per_iter=launches, num_corr=int(corr))
        n_src = frame.n
        bytes_iter = n_src * (12 + 4) + res["projective"]["num_corr"] * 24
        sec = res["projective"]["iter_ms"] * 1e-3
        rows.append(dict(frame=f"{w}x{h}", model_points=int(model.n), frame_points=int(n_src),
                         build_ms=float(np.median(build[1:])), projective=res["projective"], kdtree=res["kdtree"],
                         bytes_per_iter=int(bytes_iter), gbps=bytes_iter / sec / 1e9,
                         share_of_hbm=bytes_iter / sec / HBM_BPS))
    ctx.close()
    print(json.dumps({"gpu": name, "power_limit_w": power, "iters": args.iters, "results": rows}))


if __name__ == "__main__":
    main()
