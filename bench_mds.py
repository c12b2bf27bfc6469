"""Classical multidimensional scaling on the device (cb_vectors_mds): time per call, product passes per call, the
product kernel's time per pass against the bytes of one pass over half the matrix, and a CPU arm.

    python bench_mds.py [--repeats 3]

Workloads: n = 4 096, 16 384 and 32 768 squared Euclidean distances of seeded 16-D points with spreads 16, 15, ..., 1,
built on the device with torch; max_dim = 3 (an 8-column block, one 8-wide product per pass) and max_dim = 10 (a
16-column block). One pass of the product reads the lower triangle once: 4 n (n + 1) / 2 bytes, set against NVIDIA's
H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s (a data-sheet figure, not a measurement). Kernel times come from
torch.profiler with CUDA activities in a profiled call of its own; `call_ms` is the median host-clock time of the
synchronous call with the profiler off. Parity: the eigenvalues against those of the centred points' 16 x 16 scatter
matrix in float64 (relative 1e-4: the fp32 rounding of the entries). CPU arm, labelled as such: float64
scipy.sparse.linalg.eigsh on the explicitly formed B at n = 4 096 (the reference itself needs Eigen and Spectra).
Prints one JSON line; writes nothing."""
import argparse
import json
import subprocess
import sys
import time

import numpy as np

from cilantro_b200 import capi

HBM_BPS = 3.35e12
SIZES = [4096, 16384, 32768]
MAX_DIMS = [3, 10]
CPU_N = 4096
PRODUCT = "mds_product_kernel"


def gpu_info():
    """(name, power limit W) of GPU 0, read with nvidia-smi."""
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=60, check=True).stdout
    name, power = [x.strip() for x in out.strip().splitlines()[0].split(",")]
    return name, float(power)


def points(n, seed):
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    spread = torch.arange(16, 0, -1, device="cuda", dtype=torch.float64)
    return torch.randn(n, 16, device="cuda", generator=g, dtype=torch.float64) * spread


def squared_distances(p):
    """n x n fp32 squared distances, formed in float64 row block by row block."""
    import torch

    n = p.shape[0]
    g = (p * p).sum(1)
    out = torch.empty(n, n, device="cuda", dtype=torch.float32)
    for i in range(0, n, 4096):
        q = p[i:i + 4096]
        out[i:i + 4096] = (g[i:i + 4096, None] + g[None, :] - 2.0 * q @ p.T).clamp_min(0).to(torch.float32)
    return out


def kernel_stats(fn):
    """(product launches, product device ms, all library kernels' device ms) of one call, from torch.profiler."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    count, prod_ms, all_ms = 0, 0.0, 0.0
    for e in prof.events():
        if e.device_type != DeviceType.CUDA or "mds_" not in e.name:
            continue
        ms = e.time_range.elapsed_us() / 1e3
        all_ms += ms
        if PRODUCT in e.name:
            count += 1
            prod_ms += ms
    return count, prod_ms, all_ms


def timed(fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def cpu_arm(p):
    """float64 scipy eigsh (largest magnitude) on the explicitly formed B of the same squared distances."""
    from scipy.sparse.linalg import eigsh

    x = p.cpu().numpy()
    g = (x * x).sum(1)
    e = np.maximum(g[:, None] + g[None, :] - 2 * x @ x.T, 0).astype(np.float32).astype(np.float64)
    t0 = time.perf_counter()
    r, c, m = e.mean(1), e.mean(0), e.mean()
    B = -0.5 * (e - r[:, None] - c[None, :] + m)
    w = eigsh(B, k=3, which="LM", return_eigenvectors=True)[0]
    return (time.perf_counter() - t0) * 1e3, np.sort(w)[::-1]


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    name, power = gpu_info()
    ctx = capi.Context(0)
    out = {"gpu": name, "power_limit_w": power, "workloads": {}}
    parity = True
    for n in SIZES:
        p = points(n, seed=n)
        dm = squared_distances(p)
        torch.cuda.synchronize()  # the library copies on its own stream
        v = capi.Vectors(ctx, device_ptr=dm.data_ptr(), n=n, D=n)
        pc = (p - p.mean(0)).cpu().numpy()
        want = np.sort(np.linalg.eigvalsh(pc.T @ pc))[::-1]
        for max_dim in MAX_DIMS:
            r = capi.mds(ctx, v, max_dim)
            good = bool(r["ok"] and np.allclose(r["eigenvalues"], want[:max_dim], rtol=1e-4, atol=0))
            parity &= good
            call_ms = timed(lambda: capi.mds(ctx, v, max_dim), a.repeats)
            passes, prod_ms, all_ms = kernel_stats(lambda: capi.mds(ctx, v, max_dim))
            width = 8 if max_dim <= 6 else 16
            bytes_pass = 4.0 * n * (n + 1) / 2
            rec = {"n": n, "max_dim": max_dim, "block_columns": width, "call_ms": round(call_ms, 3),
                   "product_launches_per_call": passes, "kernel_ms_total": round(all_ms, 3),
                   "bytes_per_half_pass": bytes_pass, "parity_float64": good,
                   "eigenvalues": [float(x) for x in r["eigenvalues"]],
                   "scatter_eigenvalues_float64": [float(x) for x in want[:max_dim]]}
            if passes:
                per = prod_ms / passes
                rec["product_ms_per_pass"] = round(per, 4)
                rec["product_share_of_hbm"] = round(bytes_pass / HBM_BPS / (per * 1e-3), 3)
            else:
                rec["note"] = "the product kernel did not show in the profiler trace"
            out["workloads"][f"n{n}_dim{max_dim}"] = rec
        if n == CPU_N:
            ms, w = cpu_arm(p)
            out["cpu_scipy_eigsh_float64_explicit_B"] = {"n": n, "k": 3, "ms": round(ms, 1),
                                                         "eigenvalues": [float(x) for x in w]}
        v.close()
        del dm, p
        torch.cuda.empty_cache()
    ctx.close()
    out["parity"] = parity
    print(json.dumps(out))
    return 0 if parity else 1


if __name__ == "__main__":
    sys.exit(main())
