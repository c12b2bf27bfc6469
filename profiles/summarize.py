#!/usr/bin/env python
"""Turn the ncu captures in captures/ (tools/ncu_capture.sh) into the committed summaries of this directory.

    python profiles/summarize.py r01        # reads captures/prof_r01*.ncu-rep, captures/launches_r01.csv

Writes profiles/<round>_<kernel>.md (key metrics + top stall reasons + opcode mix of one launch),
profiles/launches_<round>.csv (copied) + a launch-share table, and profiles/traffic.json (DRAM bytes per
launch of the dominant kernel, read by bench.py for roofline.traffic).
"""
import collections
import csv
import json
import os
import re
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "captures")

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "launch__grid_size",
    "launch__block_size", "launch__registers_per_thread", "launch__shared_mem_per_block_static",
    "launch__shared_mem_per_block_dynamic", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "smsp__issue_active.avg.per_cycle_active", "smsp__warps_eligible.avg.per_cycle_active",
    "smsp__inst_executed.sum", "sass__thread_inst_executed_per_opcode_category",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct", "l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum",
    "TPC.TriageCompute.sm__cycles_active.avg", "sm__cycles_elapsed.max",
]
UNIT = {"Mbyte": 1e6, "Kbyte": 1e3, "Gbyte": 1e9, "byte": 1.0}


def ncu_csv(rep, page, extra=()):
    out = subprocess.run(["ncu", "-i", rep, "--page", page, "--csv", *extra], capture_output=True, text=True).stdout
    return list(csv.reader(out.splitlines()))


def summarize(rep, title, note):
    raw = ncu_csv(rep, "raw")
    hdr, units, row = raw[0], raw[1], raw[-1]
    col = {h: i for i, h in enumerate(hdr)}
    lines = [f"# {title}", "", note, "", f"Capture: `{os.path.basename(rep)}` (ncu --set full --clock-control none --import-source on, one launch).",
             "Numbers under the profiler are NOT bench values.", "", "| metric | value | unit |", "|---|---:|---|"]
    for k in KEYS:
        if k in col and row[col[k]] != "":
            lines.append(f"| `{k}` | {row[col[k]]} | {units[col[k]]} |")
    stalls = []
    for h, i in col.items():
        if "issue_stalled" in h and h.endswith("per_issue_active.ratio"):
            try:
                stalls.append((float(row[i]), h.replace("smsp__average_warps_issue_stalled_", "").replace("_per_issue_active.ratio", "")))
            except ValueError:
                pass
    stalls.sort(reverse=True)
    lines += ["", "Top warp-stall reasons (warps per issue-active cycle):", "", "| stall | ratio |", "|---|---:|"]
    lines += [f"| {n} | {v:.2f} |" for v, n in stalls[:8]]
    # opcode mix
    src = ncu_csv(rep, "source")
    hi = [i for i, r in enumerate(src) if "Instructions Executed" in r]
    if hi:
        h = src[hi[0]]
        ci, si, ti = h.index("Instructions Executed"), h.index("Source"), h.index("Thread Instructions Executed")
        agg = collections.defaultdict(lambda: [0, 0])
        tot = 0
        for r in src[hi[0] + 1:]:
            try:
                n, t = int(r[ci]), int(r[ti])
            except (ValueError, IndexError):
                continue
            m = re.match(r"(@!?U?P\d+\s+)?([A-Z0-9_.]+)", r[si].strip())
            op = m.group(2).split(".")[0] if m else "?"
            agg[op][0] += n
            agg[op][1] += t
            tot += n
        lines += ["", f"Executed warp-instructions by opcode (total {tot}):", "", "| opcode | warp-instr | share | active threads / instr |",
                  "|---|---:|---:|---:|"]
        for op, v in sorted(agg.items(), key=lambda x: -x[1][0])[:14]:
            lines.append(f"| {op} | {v[0]} | {100 * v[0] / max(tot, 1):.1f}% | {v[1] / max(v[0], 1):.1f} |")
    traffic = None
    if "dram__bytes_read.sum" in col:
        traffic = float(row[col["dram__bytes_read.sum"]]) * UNIT.get(units[col["dram__bytes_read.sum"]], 1.0) + \
            float(row[col["dram__bytes_write.sum"]]) * UNIT.get(units[col["dram__bytes_write.sum"]], 1.0)
        lines += ["", f"DRAM traffic of this launch: {traffic / 1e6:.1f} MB."]
    return "\n".join(lines) + "\n", traffic


def launches(csv_path):
    rows = [l for l in open(csv_path) if not l.startswith("==")]
    agg = collections.defaultdict(lambda: [0, 0.0])
    for r in csv.DictReader(rows):
        k = r["Kernel Name"].split("(")[0][-70:]
        agg[k][0] += 1
        agg[k][1] += float(r["Metric Value"].replace(",", ""))
    tot = sum(v[1] for v in agg.values())
    out = ["| launches | total us | share | avg us | kernel |", "|---:|---:|---:|---:|---|"]
    for k, v in sorted(agg.items(), key=lambda x: -x[1][1]):
        out.append(f"| {v[0]} | {v[1] / 1e3:.1f} | {100 * v[1] / tot:.1f}% | {v[1] / v[0] / 1e3:.1f} | `{k}` |")
    return "\n".join(out)


def downsample_launches(csv_path, out_path, rnd):
    """One cb_cloud_grid_downsample call (the last one of the run): time and DRAM bytes per kernel."""
    rows = list(csv.DictReader([l for l in open(csv_path) if not l.startswith("==")]))
    start = max(int(r["ID"]) for r in rows if "bin_key_kernel" in r["Kernel Name"])
    agg = collections.defaultdict(lambda: [0, 0.0, 0.0])
    for r in rows:
        if int(r["ID"]) < start:
            continue
        k = r["Kernel Name"].split("(")[0].split("::")[-1]
        v = float(r["Metric Value"].replace(",", ""))
        if r["Metric Name"] == "gpu__time_duration.sum":
            agg[k][0] += 1
            agg[k][1] += v / 1e3
        else:
            agg[k][2] += v * UNIT.get(r["Metric Unit"], 1.0)
    tot = sum(v[1] for v in agg.values())
    lines = [f"# Launches of one `cb_cloud_grid_downsample` call ({rnd}) — bench.py downsample_10m", "",
             "10 M uniform points, bin 0.01 -> 999 951 bins. `ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,"
             "dram__bytes_write.sum --clock-control none` (serialised, cold cache: compare shares).", "",
             "| kernel | launches | us | share | DRAM MB |", "|---|---:|---:|---:|---:|"]
    for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        lines.append(f"| `{k}` | {v[0]} | {v[1]:.1f} | {100 * v[1] / tot:.1f}% | {v[2] / 1e6:.1f} |")
    lines.append(f"| total | {sum(v[0] for v in agg.values())} | {tot:.1f} | 100% | {sum(v[2] for v in agg.values()) / 1e6:.1f} |")
    open(out_path, "w").write("\n".join(lines) + "\n")


def main():
    rnd = sys.argv[1] if len(sys.argv) > 1 else "r02"
    dl = os.path.join(OUT, f"launches_downsample_{rnd}.csv")
    if os.path.exists(dl):
        downsample_launches(dl, os.path.join(HERE, f"{rnd}_downsample_launches.md"), rnd)
        print("wrote downsample launches")
    flush = "L2 flushed before the iteration (as in bench.py's value leg)."
    # (report, summary file, title, note, traffic key = (workload, regime part))
    jobs = [
        (f"{rnd}_icp_cold_p2p_1m.ncu-rep", f"{rnd}_icp_search_kernel_cold_p2p_1m.md",
         "icp_search_kernel<p2p> - first iteration of an estimate() call, 1 M -> 1 M",
         "Every query is searched (nothing cached): transform + warp-pooled WIDE grid 1-NN (exclusion bound for the cache) + "
         "pivoted Kabsch moments + block/grid reduction. " + flush, ("icp_p2p_1m", "first_iteration", "search")),
        (f"{rnd}_icp_cached_p2p_1m.ncu-rep", f"{rnd}_icp_cached_pipe_kernel_p2p_1m.md",
         "icp_cached_pipe_kernel<p2p> - cached pass (with its searches) of a converged iteration, 1 M -> 1 M",
         "Per query: point + cache streamed, cached match gathered (cp.async pipeline through shared memory), exclusion test, "
         "moments of the pairs that pass; the rest searched by the warp that flagged them. " + flush, ("icp_p2p_1m", "converged_iteration", "cached")),
        (f"{rnd}_icp_finish_p2p_1m.ncu-rep", f"{rnd}_icp_finish_kernel_p2p_1m.md",
         "icp_finish_kernel<p2p> - exchange + solve, one warp", "Totals -> (peer all-reduce when world > 1) -> Kabsch, rotation(), "
         "compose, convergence test -> LoopState.", ("icp_p2p_1m", "converged_iteration", "finish")),
        (f"{rnd}_icp_cold_combined_10m.ncu-rep", f"{rnd}_icp_search_kernel_cold_combined_10m.md",
         "icp_search_kernel<combined> - first iteration, 10 M -> 10 M (BASELINE config 3 on one GPU)",
         "As above with the 28-value Gauss-Newton normal equations (point + plane terms). " + flush,
         ("icp_combined_10m", "first_iteration", "search")),
        (f"{rnd}_icp_cached_combined_10m.ncu-rep", f"{rnd}_icp_cached_pipe_kernel_combined_10m.md",
         "icp_cached_pipe_kernel<combined> - cached pass of a converged iteration, 10 M -> 10 M",
         "560 MB algorithmic (16 B point + 8 B cache + 16 B match + 16 B normal per query). " + flush,
         ("icp_combined_10m", "converged_iteration", "cached")),
        (f"{rnd}_kmeans_50m.ncu-rep", f"{rnd}_kmeans_assign_kernel.md", "kmeans_assign_kernel - bench.py kmeans_50m (BASELINE config 4)",
         "50 M points x 1024 centroids, the shipped kernel with its occupancy-sized persistent grid: fused assignment + "
         "per-cluster double sums (shared-memory atomics).", None),
        (f"{rnd}_ransac_5m.ncu-rep", f"{rnd}_ransac_score_kernel.md", "ransac_score_kernel - bench.py ransac_5m (BASELINE config 5)",
         "5 M correspondences x 1000 hypotheses per launch, inlier counts only.", None),
    ]
    traffic = {}
    for rep, md, title, note, key in jobs:
        p = os.path.join(OUT, rep)
        if not os.path.exists(p):
            continue
        text, tr = summarize(p, title, note)
        open(os.path.join(HERE, md), "w").write(text)
        if key and tr:
            w, regime, part = key
            traffic.setdefault(w, {}).setdefault(regime, {})[part] = tr
        print("wrote", md)
    for w, regs in traffic.items():
        for regime in list(regs):
            regs[regime]["total"] = sum(v for k, v in regs[regime].items() if k != "total")
    traffic["source"] = f"profiles/{rnd}_icp_*.md (ncu --set full, dram__bytes_read.sum + dram__bytes_write.sum per launch)"
    json.dump(traffic, open(os.path.join(HERE, "traffic.json"), "w"), indent=1)
    lp = os.path.join(OUT, f"launches_{rnd}.csv")
    if os.path.exists(lp):
        shutil.copy(lp, os.path.join(HERE, f"launches_{rnd}.csv"))
        open(os.path.join(HERE, f"launches_{rnd}.md"), "w").write(
            f"# Launch list of one `bench.py --no-secondary --no-cpu-baseline` run ({rnd})\n\n`ncu --metrics gpu__time_duration.sum "
            "--clock-control none` - cold-cache, serialised: compare SHARES, not absolutes. The run contains the grid builds, the\n"
            "warm-up and timed estimate() calls of both poses, the clock-sampler filler iterations and three end-to-end calls.\n\n"
            + launches(lp) + "\n")
        print("wrote launches")


if __name__ == "__main__":
    main()
