"""Depth-image and RGB-D <-> cloud conversions on the device (cb_depth_image_to_points, cb_points_to_depth_image,
cb_points_to_index_map): device time per call, the same with the raw frame's host -> device copy, bytes moved over
kernel time, and launches per call.

    python bench_depth_images.py [--repeats 20]

Workloads: 640 x 480, 1920 x 1080 and 8192 x 8192 uint16 depth frames of a smooth seeded surface with 20 % holes and an
RGB frame of the same size, intrinsics of a 525 px pinhole scaled to the width. Legs per size: depth -> points,
depth -> points + normals, RGB-D -> points + normals + colours (each compacting, output to a device Cloud so no
device -> host copy is timed), and cloud -> depth image / index map of the frame's own points (host images out). The
"device" time feeds a frame already in device memory (a torch CUDA tensor); the "with copy" time passes the host frame,
so the call includes its upload. `call_ms` are medians of CUDA-event-bracketed calls, which include the outputs'
allocation and, for host outputs, their device -> host copies; `kernel_ms` is the device time of the library's kernels
in one call of its own under torch.profiler. Bytes are the minimum each leg must move in HBM (raw frame read, flags and
scan, outputs written; for rendering, points read, the 8 B z-buffer word read and the image written), over kernel
time, set against NVIDIA's H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s (a data-sheet figure, not a measurement). Prints one JSON line; writes nothing."""
import argparse
import json
import subprocess

import numpy as np

from cilantro_b200 import capi

HBM_BPS = 3.35e12
SIZES = [(640, 480), (1920, 1080), (8192, 8192)]


def gpu_info():
    """(name, power limit W) of GPU 0, read with nvidia-smi."""
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=60, check=True).stdout
    name, power = [x.strip() for x in out.strip().splitlines()[0].split(",")]
    return name, float(power)


class CudaImage:
    """A torch CUDA tensor seen as a uint16 array (torch keeps the bits as int16)."""

    def __init__(self, t, dtype):
        self.t, self.shape = t, tuple(t.shape)
        self.__cuda_array_interface__ = dict(t.__cuda_array_interface__, typestr=np.dtype(dtype).str)


def frame(w, h, seed=0):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    d = (1500 + 300 * np.sin(xx * (40.0 / w)) * np.cos(yy * (30.0 / h))).astype(np.uint16)
    d[rng.random((h, w)) < 0.2] = 0
    return d, rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


KERNELS = ("depth_points_kernel", "scan_block_kernel", "scan_sums_kernel", "scan_add_kernel", "render_keys_kernel",
           "render_write_kernel")


def kernel_ms(fn):
    """Device time of the library's kernels in one call, from torch.profiler with CUDA activities."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(e.time_range.elapsed_us() / 1e3 for e in prof.events()
               if e.device_type == DeviceType.CUDA and any(k in e.name for k in KERNELS))


def timed(torch, fn, repeats):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    args = ap.parse_args()
    name, power = gpu_info()
    ctx = capi.Context(0)
    conv = capi.DepthConverter(np.uint16, 1000.0)
    rows = []
    for w, h in SIZES:
        K = np.array([[525.0 * w / 640, 0, (w - 1) / 2], [0, 525.0 * w / 640, (h - 1) / 2], [0, 0, 1]], np.float32)
        depth, rgb = frame(w, h)
        dd = CudaImage(torch.from_numpy(depth.view(np.int16)).cuda(), np.uint16)
        dr = torch.from_numpy(rgb).cuda()
        npix = w * h
        legs = {"points": dict(), "points_normals": dict(normals=True),
                "rgbd_points_normals_colors": dict(normals=True, rgb=True)}
        for leg, kw in legs.items():
            rgb_dev = dr if kw.get("rgb") else None
            rgb_host = rgb if kw.get("rgb") else None
            normals = kw.get("normals", False)
            out = {}

            def call(src, colour):
                r = capi.depth_image_to_points(ctx, src, K, conv, rgb=colour, normals=normals, to_device=True)
                out["m"] = r["count"]
                r["cloud"].close()

            l0 = ctx.kernel_launches()
            call(dd, rgb_dev)
            launches = ctx.kernel_launches() - l0
            dev = timed(torch, lambda: call(dd, rgb_dev), args.repeats)
            host = timed(torch, lambda: call(depth, rgb_host), args.repeats)
            m = out["m"]
            # raw read twice (+ rgb once), flags written and scanned (~4 x 4 B), outputs written (12 B points, 12 B
            # normals, colours go to the host: 12 B written on the device)
            b = npix * 2 * 2 + npix * 16 + m * 12 * (1 + normals) + (npix * 3 + m * 12 if kw.get("rgb") else 0)
            kms = kernel_ms(lambda: call(dd, rgb_dev))
            rows.append(dict(size=f"{w}x{h}", leg=leg, kept=m, launches=launches, call_ms=dev, with_copy_ms=host,
                             kernel_ms=kms, bytes=b, hbm_share_of_kernels=b / (kms * 1e-3) / HBM_BPS))
        pts = capi.depth_image_to_points(ctx, depth, K, conv, to_device=True)["cloud"]
        n = pts.n
        for leg, fn in (("cloud_to_depth", lambda: capi.points_to_depth_image(ctx, pts, K, w, h, conv)),
                        ("cloud_to_index_map", lambda: capi.points_to_index_map(ctx, pts, K, w, h))):
            l0 = ctx.kernel_launches()
            fn()
            launches = ctx.kernel_launches() - l0
            t = timed(torch, fn, args.repeats)
            kms = kernel_ms(fn)
            out_b = 2 if leg == "cloud_to_depth" else 8
            b = n * 12 + npix * (8 + out_b)  # the z-buffer's memset is not a kernel; its atomics stay in L2
            rows.append(dict(size=f"{w}x{h}", leg=leg, points=n, launches=launches, call_ms=t, kernel_ms=kms, bytes=b,
                             hbm_share_of_kernels=b / (kms * 1e-3) / HBM_BPS))
        pts.close()
    ctx.close()
    print(json.dumps({"gpu": name, "power_limit_w": power, "results": rows}))


if __name__ == "__main__":
    main()
