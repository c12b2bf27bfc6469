"""k-means over D-dimensional rows (cb_kmeans_*_vectors): device time of one assignment and of one Lloyd iteration
on three workloads, the FP32 operations the assignment model counts and the share of the card's non-FMA FP32 issue
rate they reach.

    python bench_kmeans_features.py [--repeats 7] [--iters 5] [--sample 20000]

Workloads: 10 M x D = 6 x K = 256 (xyz + weighted colour, the reference example's 6-D recipe at scan scale),
1 M x D = 32 x K = 1024 and 1 M x D = 128 x K = 256 (descriptor clustering; the second takes the global-sums path).
Times are CUDA-event times on the library's stream (gpu_ms_total of cb_kmeans_cluster_vectors), median over the
repeats after one warm-up run: `assign_ms` is a run with max_iter = 1 (one assignment kernel plus the per-step
centroid upload and sums download), `lloyd_iter_ms` a run of --iters iterations with tol = 0 divided by its
iterations. The model counts 3 N K D fp32 operations per assignment (subtract, multiply, add; the distance contract
forbids FMA); the peak is SMs x 128 lanes x the maximum SM clock. One assignment's labels are checked bit-exact
against the numpy restatement (tests/kmeans_features_ref.py) on a row sample. Prints one JSON line; writes nothing."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

from cilantro_b200 import capi

sys.dont_write_bytecode = True  # the restatement is imported from tests/; leave no cache in the tree
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tests"))
import kmeans_features_ref as kf  # noqa: E402

WORKLOADS = [("n10m_d6_k256", 10_000_000, 6, 256), ("n1m_d32_k1024", 1_000_000, 32, 1024),
             ("n1m_d128_k256", 1_000_000, 128, 256)]


def gpu_info():
    """(name, power limit W, max SM clock MHz) of GPU 0, read with nvidia-smi."""
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                          "-i", "0"], capture_output=True, text=True, timeout=60, check=True).stdout
    name, power, clock = [x.strip() for x in out.strip().splitlines()[0].split(",")]
    return name, float(power), float(clock)


def data(n, D, k, seed):
    """Rows around k / 4 gaussian blobs (a clustered scene, not uniform noise) and k distinct rows as seeds."""
    rng = np.random.default_rng(seed)
    centres = rng.uniform(-1, 1, (max(1, k // 4), D)).astype(np.float32)
    pts = centres[rng.integers(0, len(centres), n)]
    pts += rng.normal(0, 0.15, (n, D)).astype(np.float32)
    return pts, pts[rng.choice(n, k, replace=False)].copy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--sample", type=int, default=20000)
    a = ap.parse_args()

    name, power, clock_mhz = gpu_info()
    ctx = capi.Context(0)
    sms = ctx.device_info()["sm_count"]
    peak = sms * 128 * clock_mhz * 1e6  # non-FMA fp32 operations per second
    out = {"gpu": name, "power_limit_w": power, "sm_count": sms, "max_sm_clock_mhz": clock_mhz, "workloads": {}}
    parity = True
    for tag, n, D, k in WORKLOADS:
        pts, cent0 = data(n, D, k, seed=D)
        v = capi.Vectors(ctx, pts)
        labels, _, _ = capi.kmeans_assign(ctx, v, cent0)
        rows = np.random.default_rng(1).choice(n, min(a.sample, n), replace=False)
        ok = bool(np.array_equal(labels[rows], kf.assign(pts[rows], cent0)))
        parity &= ok

        def run(max_iter):
            r = capi.kmeans_cluster(ctx, v, cent0, max_iter=max_iter, tol=0.0, want_labels=False)
            return r["gpu_ms_total"], r["iterations"]

        run(1)
        assign_ms = float(np.median([run(1)[0] for _ in range(a.repeats)]))
        its = [run(a.iters) for _ in range(a.repeats)]
        iter_ms = float(np.median([ms / it for ms, it in its]))
        ops = 3.0 * n * k * D
        out["workloads"][tag] = {
            "n": n, "D": D, "k": k, "assign_ms": round(assign_ms, 4), "lloyd_iter_ms": round(iter_ms, 4),
            "lloyd_iterations": int(its[0][1]), "model_fp32_ops": ops,
            "achieved_tflops": round(ops / (assign_ms * 1e-3) / 1e12, 2),
            "share_of_fp32_issue": round(ops / (assign_ms * 1e-3) / peak, 3),
            "ideal_assign_ms": round(ops / peak * 1e3, 4), "labels_bitexact_on_sample": ok,
        }
        v.close()
    ctx.close()
    out["parity"] = parity
    print(json.dumps(out))
    return 0 if parity else 1


if __name__ == "__main__":
    sys.exit(main())
