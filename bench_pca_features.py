"""Covariance and PCA projection over D-dimensional rows (cb_vectors_mean_cov, cb_vectors_project): device time per
kernel, host-clock call time, the host eigen-solve time, the model's bytes and FP64 operations, and the share of the
larger data-sheet bound.

    python bench_pca_features.py [--repeats 7]

Workloads: 10 M x 6 (xyz + colour features at scan scale; HBM-bound), 10 M x 32, 1 M x 128 and 1 M x 512 covariance
(descriptor widths; the last is FP64-bound), and a 10 M x 32 -> 8 projection. The covariance model counts 4 n D bytes
read and n D (D + 1) FP64 operations (the upper triangle of the rank-n update, one multiply and one add per entry);
the projection model 4 n (D + k) bytes and 2 n D k FP32 operations. The bounds are NVIDIA's H100 SXM data-sheet
figures, not measurements: 3.35 TB/s HBM3, 67 TFLOP/s FP64 tensor (the covariance kernel runs on DMMA) and 67 TFLOP/s
FP32 with FMA, so 33.5 TFLOP/s for the projection's separate multiplies and adds. The share is the larger of the two model times over the measured kernel time, with the bound that set it.
Kernel times come from torch.profiler with CUDA activities, in a profiled pass of its own; `call_ms` is the median
host-clock time of the synchronous call with the profiler off; `eigen_ms` the host time of cb_solve_sym_eigen on the
returned covariance. Parity: the covariance is checked against float64 (DESIGN §4.18 bound) and the projection bit
for bit against the restatement on a row sample. Prints one JSON line; writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

from cilantro_b200 import capi

sys.dont_write_bytecode = True  # the restatement is imported from tests/; leave no cache in the tree
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tests"))
import pca_features_ref as pf  # noqa: E402

HBM_BPS = 3.35e12
FP64_TENSOR = 67e12
FP32_NO_FMA = 67e12 / 2  # the projection's contract forbids FMA: one multiply and one add issue separately
COV_WORKLOADS = [("cov_n10m_d6", 10_000_000, 6), ("cov_n10m_d32", 10_000_000, 32), ("cov_n1m_d128", 1_000_000, 128),
                 ("cov_n1m_d512", 1_000_000, 512)]
PROJ_WORKLOAD = ("project_n10m_d32_k8", 10_000_000, 32, 8)
KERNELS = ("cov_pivot_kernel", "cov_accumulate_kernel", "cov_fold_kernel", "pca_map_kernel")


def gpu_info():
    """(name, power limit W) of GPU 0, read with nvidia-smi."""
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=60, check=True).stdout
    name, power = [x.strip() for x in out.strip().splitlines()[0].split(",")]
    return name, float(power)


def data(n, D, seed):
    """Rows with per-dimension offsets and scales and some correlation (a low-rank part plus noise)."""
    rng = np.random.default_rng(seed)
    r = max(1, D // 4)
    mix = rng.standard_normal((r, D)).astype(np.float32)
    out = np.empty((n, D), np.float32)
    step = 1_000_000
    for i in range(0, n, step):
        m = min(step, n - i)
        out[i:i + m] = rng.standard_normal((m, r), dtype=np.float32) @ mix
        out[i:i + m] += rng.standard_normal((m, D), dtype=np.float32) * 0.3
    out *= rng.uniform(0.5, 4, D).astype(np.float32)
    out += rng.uniform(-100, 100, D).astype(np.float32)
    return out


def float64_mean_cov(rows):
    """Two-pass float64 mean and covariance, in row blocks."""
    n, D = rows.shape
    step = 1_000_000
    s = np.zeros(D)
    for i in range(0, n, step):
        s += rows[i:i + step].astype(np.float64).sum(0)
    mean = s / n
    c = np.zeros((D, D))
    for i in range(0, n, step):
        x = rows[i:i + step].astype(np.float64) - mean
        c += x.T @ x
    return mean, c / (n - 1)


def kernel_times(calls):
    """{tag: {kernel: device ms}} of one call of each fn in calls {tag: fn}, in one torch.profiler session with CUDA
    activities. The calls are synchronous, so a kernel belongs to the tagged range it ran inside."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile, record_function

    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], acc_events=True) as prof:
        for tag, fn in calls.items():
            with record_function("bench:" + tag):
                fn()
        torch.cuda.synchronize()
    evs = prof.events()
    ranges = {e.name[6:]: (e.time_range.start, e.time_range.end) for e in evs if e.name.startswith("bench:")}
    times = {tag: {} for tag in calls}
    for e in evs:
        if e.device_type != DeviceType.CUDA:
            continue
        k = next((k for k in KERNELS if k in e.name), None)
        if k is None:
            continue
        for tag, (t0, t1) in ranges.items():
            if t0 <= e.time_range.start <= t1:
                times[tag][k] = times[tag].get(k, 0.0) + e.time_range.elapsed_us() / 1e3
    return times


def timed(fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def share(bytes_, flops, peak_flops, ms):
    t_mem, t_flop = bytes_ / HBM_BPS, flops / peak_flops
    return round(max(t_mem, t_flop) / (ms * 1e-3), 3), ("HBM" if t_mem >= t_flop else "compute")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    a = ap.parse_args()

    name, power = gpu_info()
    ctx = capi.Context(0)
    out = {"gpu": name, "power_limit_w": power, "workloads": {}}
    parity = True
    sets = {}  # tag: (device set, the call, its main kernel, its compute peak)
    for tag, n, D in COV_WORKLOADS:
        rows = data(n, D, seed=D)
        v = capi.Vectors(ctx, rows)
        mean, cov, ok = capi.mean_cov(ctx, v)
        rm, rc = float64_mean_cov(rows)
        good = bool(ok and pf.within_cov_bound(mean, cov, rm, rc))
        parity &= good
        call_ms = timed(lambda v=v: capi.mean_cov(ctx, v), a.repeats)
        covd = cov.astype(np.float64)
        eig_ms = timed(lambda: capi.solve_sym_eigen(covd), 3)
        out["workloads"][tag] = {"n": n, "D": D, "call_ms": round(call_ms, 4), "eigen_ms": round(eig_ms, 3),
                                 "model_bytes": 4.0 * n * D, "model_fp64_ops": float(n) * D * (D + 1),
                                 "parity_float64": good}
        sets[tag] = (v, lambda v=v: capi.mean_cov(ctx, v), "cov_accumulate_kernel", FP64_TENSOR)
        del rows

    tag, n, D, k = PROJ_WORKLOAD
    rows = data(n, D, seed=D + 1)
    v = capi.Vectors(ctx, rows)
    r = capi.pca(ctx, v)
    proj = capi.pca_project(ctx, v, r["mean"], r["eigenvectors"], k)
    sample = np.random.default_rng(1).choice(n, 20000, replace=False)
    good = bool(np.array_equal(proj[sample], pf.project(rows[sample], r["mean"], r["eigenvectors"], k), equal_nan=True))
    parity &= good
    call_ms = timed(lambda: capi.pca_project(ctx, v, r["mean"], r["eigenvectors"], k, to_device=True).close(),
                    a.repeats)
    out["workloads"][tag] = {"n": n, "D": D, "k": k, "call_ms": round(call_ms, 4), "model_bytes": 4.0 * n * (D + k),
                             "model_fp32_ops": 2.0 * n * D * k, "bitexact_on_sample": good}
    sets[tag] = (v, lambda: capi.pca_project(ctx, v, r["mean"], r["eigenvectors"], k, to_device=True).close(),
                 "pca_map_kernel", FP32_NO_FMA)
    del rows

    for _, fn, _, _ in sets.values():  # warm every call of the profiled pass
        fn()
    kt = kernel_times({tag: fn for tag, (_, fn, _, _) in sets.items()})
    for tag, (v, _, main_kernel, peak) in sets.items():
        rec = out["workloads"][tag]
        rec["kernel_ms"] = {x: round(t, 4) for x, t in kt[tag].items()}
        ops = rec.get("model_fp64_ops", rec.get("model_fp32_ops"))
        if kt[tag].get(main_kernel):
            rec["share"], rec["bound"] = share(rec["model_bytes"], ops, peak, kt[tag][main_kernel])
        else:
            rec["note"] = "the library's kernels did not show in the profiler trace; call_ms is the host-clock time"
        v.close()
    ctx.close()
    out["parity"] = parity
    print(json.dumps(out))
    return 0 if parity else 1


if __name__ == "__main__":
    sys.exit(main())
