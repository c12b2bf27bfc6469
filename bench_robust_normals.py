"""Robust (MCD) normal estimation: device time at 1 M points, k = 12, for the reference example's recipe
(2 trials, 1 refinement, chi-square 6.25) and the reference's defaults (6 trials, 3 refinements), next to plain
normals on the same cloud; and the serial oracle's CPU time at 100 k points for scale.

    python bench_robust_normals.py [--n 1000000] [--k 12] [--repeats 10] [--oracle-n 100000]

Prints one JSON line. Device times are CUDA-event times of the kernels (gpu_ms of the C ABI), median over the repeats
after one warm-up call each. Writes nothing."""
import argparse
import json
import subprocess
import time

import numpy as np

from cilantro_b200 import capi, synth

RECIPE = dict(num_trials=2, num_refinements=1, chi_square_threshold=6.25)
DEFAULTS = dict(num_trials=6, num_refinements=3)


def scene(n, seed=1):
    """A scanned sheet with 10 % of the points pushed 1-3 cm off it."""
    pts, nrm = synth.surface_cloud(n, seed=seed, noise=0.0005)
    rng = np.random.default_rng(seed)
    off = rng.random(n) < 0.1
    pts[off] += (nrm[off] * rng.uniform(0.01, 0.03, (off.sum(), 1))).astype(np.float32)
    return pts


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--k", type=int, default=12)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--oracle-n", type=int, default=100_000)
    a = ap.parse_args()

    ctx = capi.Context(0)
    cloud = capi.Cloud(ctx, scene(a.n))
    runs = {"plain": lambda: cloud.estimate_normals(k=a.k, fetch=False)["gpu_ms"],
            "mcd_recipe": lambda: cloud.estimate_normals_mcd(k=a.k, seed=1, fetch=False, **RECIPE)["gpu_ms"],
            "mcd_defaults": lambda: cloud.estimate_normals_mcd(k=a.k, seed=1, fetch=False, **DEFAULTS)["gpu_ms"]}
    ms = {}
    for name, fn in runs.items():
        fn()
        ms[name] = float(np.median([fn() for _ in range(a.repeats)]))
    invalid = int((cloud.estimate_normals_mcd(k=a.k, seed=1, **RECIPE)["status"] != 0).sum())
    ctx.close()

    from scipy.spatial import cKDTree

    from oracle import robust_normals as orn

    small = scene(a.oracle_n, seed=2)
    _, idx = cKDTree(small).query(small, a.k)
    cnt = np.full(a.oracle_n, a.k, np.uint32)
    oracle_ms = {}
    for name, kw in (("mcd_recipe", RECIPE), ("mcd_defaults", DEFAULTS)):
        t0 = time.perf_counter()
        orn.estimate_normals_mcd(small, k=a.k, seed=1, neighbors=(idx, cnt), **kw)
        oracle_ms[name] = (time.perf_counter() - t0) * 1e3

    print(json.dumps({"workload": "robust_normals", "gpu": gpu_info(), "n": a.n, "k": a.k,
                      "device_ms": {key: round(v, 3) for key, v in ms.items()}, "recipe_invalid": invalid,
                      "oracle_cpu_ms": {"n": a.oracle_n, **{key: round(v, 1) for key, v in oracle_ms.items()}}}))


if __name__ == "__main__":
    main()
