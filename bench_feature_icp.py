"""Feature-space rigid ICP (cb_icp_set_features): per-iteration device time at 1 M -> 1 M points on the textured sheet
(synth.textured_sheet_pair) for each feature kind, next to the default path on the same pair (device-resident loop) and
the list path with point-only features (inlier fraction 0.999, a non-default engine option), which separates the cost of
the features from the cost of the list path; per feature kind, how many destination points lie inside the xyz ball a
query must scan (xyz_ball_points, counted on the CPU for a sample of queries under the final transform); and, for
scale, the CPU time of the reference's own nanoflann feature search (oracle/_ref, where it was built) at --ref-n points.

    python bench_feature_icp.py [--n 1000000] [--iters 10] [--ref-n 100000]

Prints one JSON line. Device times are the per-iteration CUDA-event brackets of cb_icp_estimate (timing = 1: the
iteration's kernels, the reduction and the host solve), median over the iterations after one warm-up estimate. Combined
metric (w_pt 0.1, w_pl 1), max_d2 0.05, weights w_n 0.5, w_c 5 (the reference example's recipe). Writes nothing."""
import argparse
import json
import subprocess
import time

import numpy as np

from cilantro_b200 import capi, synth

W_N, W_C = 0.5, 5.0
KW = dict(metric="combined", w_pt=0.1, w_pl=1.0, tol=0.0, max_d2=0.05, timing=1)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def arrays(kind, s):
    nrm, col = "normal" in kind, "color" in kind
    return dict(dst_normals=s["dst_normals"] if nrm else None, dst_colors=s["dst_colors"] if col else None,
                src_normals=s["src_normals"] if nrm else None, src_colors=s["src_colors"] if col else None)


def xyz_ball_points(kind, s, T, sample=2000):
    """Points of the destination inside the xyz ball of radius sqrt(best feature d2) around each of `sample` source
    queries under T (median, mean): the candidates every exact search that prunes on the xyz part alone must evaluate.
    Counted on the CPU with scipy kd-trees (float64)."""
    from scipy.spatial import cKDTree

    def feats(p, n, c):
        parts = [p]
        if "normal" in kind:
            parts.append(W_N * n)
        if "color" in kind:
            parts.append(W_C * c)
        return np.hstack(parts).astype(np.float64)

    rng = np.random.default_rng(0)
    pick = rng.choice(s["src"].shape[0], sample, replace=False)
    R, t = T[:, :3].astype(np.float64), T[:, 3].astype(np.float64)
    q = s["src"][pick] @ R.T + t
    qf = feats(q, s["src_normals"][pick] @ R.T, s["src_colors"][pick])
    best, _ = cKDTree(feats(s["dst"], s["dst_normals"], s["dst_colors"])).query(qf, k=1)
    inside = best ** 2 < KW["max_d2"]
    counts = cKDTree(s["dst"].astype(np.float64)).query_ball_point(q, np.where(inside, best, np.sqrt(KW["max_d2"])),
                                                                    return_length=True)
    return {"median": float(np.median(counts)), "mean": float(np.mean(counts)), "queries": sample}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--ref-n", type=int, default=100_000)
    a = ap.parse_args()

    s = synth.textured_sheet_pair(a.n, seed=1)
    ctx = capi.Context(0)
    dst, src = capi.Cloud(ctx, s["dst"], s["dst_normals"]), capi.Cloud(ctx, s["src"])
    runs = {"default_path": ("point", {}), "list_path_point": ("point", dict(inlier_fraction=0.999))}
    for kind in ("point_normal", "point_color", "point_normal_color"):
        runs[kind] = (kind, {})
    out = {"metric": "feature_icp_ms_per_iter", "n": a.n, "gpu": gpu_info(), "max_d2": KW["max_d2"], "w_n": W_N,
           "w_c": W_C}
    for name, (kind, extra) in runs.items():
        icp = capi.Icp(ctx, dst, src)
        if kind != "point":
            icp.set_features(kind, normal_weight=W_N, color_weight=W_C, **arrays(kind, s))
        icp.estimate(max_iter=2, **KW, **extra)  # warm-up
        r = icp.estimate(max_iter=a.iters, **KW, **extra)
        out[name] = {"ms_per_iter": float(np.median(r["iter_ms"])), "num_corr": r["num_corr"],
                     "offset_error": float(np.linalg.norm(r["T"][:2, 3] - s["T_ref"][:2, 3]))}
        if kind != "point":
            out[name]["xyz_ball_points"] = xyz_ball_points(kind, s, r["T"])
        icp.close()
    ctx.close()

    from oracle import feature_icp

    if feature_icp.have_ref():
        m = min(a.ref_n, a.n)
        dt = feature_icp.tails("point_normal_color", s["dst_normals"][:m], s["dst_colors"][:m], W_N, W_C)
        st = feature_icp.tails("point_normal_color", s["src_normals"][:m], s["src_colors"][:m], W_N, W_C)
        fd = feature_icp.features("point_normal_color", capi.identity(), s["dst"][:m], dt)
        fs = feature_icp.features("point_normal_color", capi.identity(), s["src"][:m], st)
        t0 = time.perf_counter()
        feature_icp.ref_knn1(fd, fs, KW["max_d2"])
        out["ref_nanoflann_d9_cpu_ms"] = {"n": m, "ms": (time.perf_counter() - t0) * 1e3,
                                          "note": "tree build + one search of every query, OpenMP threads of this host"}
    else:
        out["ref_nanoflann_d9_cpu_ms"] = "not built"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
