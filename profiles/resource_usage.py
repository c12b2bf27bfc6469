"""Registers / stack / shared memory per kernel of the built library, from `cuobjdump --dump-resource-usage`
(no GPU needed). Writes profiles/resource_usage.md.   python profiles/resource_usage.py"""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "cilantro_b200", "libcilantro_b200.so")
HOT = ("icp_search_kernel", "icp_cached_pipe_kernel", "icp_finish_kernel", "icp_pass_kernel",
       "pairs_pass_kernel", "kmeans_assign_kernel", "ransac_score_kernel", "inlier_moments_kernel", "moments_kernel",
       "normals_knn_kernel", "normals_radius_kernel", "knn_k_kernel", "radius_kernel", "residual_kernel",
       "segment_kernel", "shift_kernel", "round_kernel", "rep_kernel", "plane_score_kernel", "plane_fit_kernel",
       "plane_moments_kernel", "inlier_scatter_kernel", "warp_assemble_kernel", "warp_cg_kernel", "warp_compose_kernel")


def main():
    raw = subprocess.run(["cuobjdump", "--dump-resource-usage", LIB], capture_output=True, text=True, check=True).stdout
    names = subprocess.run(["c++filt"], input=raw, capture_output=True, text=True, check=True).stdout.splitlines()
    rows, fn = [], None
    for line in names:
        m = re.match(r"\s*Function (.*):\s*$", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", line)
        if m and fn:
            short = re.sub(r"\(anonymous namespace\)::|cb::|void ", "", fn)
            short = re.sub(r"\(.*$", "", short)
            if any(h in short for h in HOT):
                rows.append((short, *map(int, m.groups())))
            fn = None
    rows = sorted(set(rows))  # kernels of a shared header (radius_lists.cuh) appear once per translation unit
    out = ["# Kernel resources (`cuobjdump --dump-resource-usage`, sm_90a)", "",
           "STACK is per-thread local memory the kernel reserves: call frames of the out-of-line far-chunk search",
           "(`search_chunk_far`, DESIGN §4.2), the k-best arrays of the general-k search, and spills. The loop's cached pass",
           "(`icp_cached_pipe_kernel`) and the k-means / RANSAC kernels stay (almost) in registers.",
           "`MODE` template values: 0 correspondences only, 1 p2p raw moments, 2 combined, 3 p2p pivoted moments.", "",
           "| kernel | registers | stack B | static smem B |", "|---|---:|---:|---:|"]
    for name, reg, stack, smem, _local in rows:
        out.append(f"| `{name}` | {reg} | {stack} | {smem} |")
    path = os.path.join(ROOT, "profiles", "resource_usage.md")
    with open(path, "w") as f:
        f.write("\n".join(out) + "\n")
    print(path, len(rows), "kernels")


if __name__ == "__main__":
    main()
