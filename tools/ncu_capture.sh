#!/usr/bin/env bash
# ncu captures for profiles/summarize.py (summaries + profiles/traffic.json); run on a GPU machine with a working
# Nsight Compute, reports land in captures/.
set -u
cd "$(dirname "$0")/.."
mkdir -p captures
NCU="ncu --set full --clock-control none --import-source on"
if [ -z "${SKIP_1M:-}" ]; then
# device-resident ICP loop, 1 M p2p: 2 estimate() calls x (1 cold search + 14 cached passes, each + 1 finish) launches
FLUSH=1 $NCU -k regex:icp_search_kernel -s 1 -c 1 -o captures/r02_icp_cold_p2p_1m python tools/loop_run.py 1000000 p2p 15 > /dev/null 2>&1
FLUSH=1 $NCU -k regex:icp_cached_pipe_kernel -s 10 -c 1 -o captures/r02_icp_cached_p2p_1m python tools/loop_run.py 1000000 p2p 15 > /dev/null 2>&1
FLUSH=1 $NCU -k regex:icp_finish_kernel -s 12 -c 1 -o captures/r02_icp_finish_p2p_1m python tools/loop_run.py 1000000 p2p 15 > /dev/null 2>&1
fi
if [ -z "${SKIP_10M:-}" ]; then
# 10 M combined
FLUSH=1 $NCU -k regex:icp_search_kernel -s 1 -c 1 -o captures/r02_icp_cold_combined_10m python tools/loop_run.py 10000000 combined 10 > /dev/null 2>&1
FLUSH=1 $NCU -k regex:icp_cached_pipe_kernel -s 7 -c 1 -o captures/r02_icp_cached_combined_10m python tools/loop_run.py 10000000 combined 10 > /dev/null 2>&1
fi
# (all of the above with the L2 flushed before every iteration, as in bench.py's value leg: FLUSH=1)
# k-means 50 M x 1024, RANSAC 5 M x 1000 (the shipped kernels on the BASELINE configs)
[ -n "${SKIP_AUX:-}" ] || $NCU -k regex:kmeans_assign_kernel -s 1 -c 1 -o captures/r02_kmeans_50m python bench.py --workload kmeans_50m --steps 2 --warmup 1 > /dev/null 2>&1
[ -n "${SKIP_AUX:-}" ] || $NCU -k regex:ransac_score_kernel -s 1 -c 1 -o captures/r02_ransac_5m python bench.py --workload ransac_5m --steps 1 --warmup 1 > /dev/null 2>&1
if [ -z "${SKIP_LAUNCHES:-}" ]; then
# every launch of one default bench run with its device time (shares)
ncu --metrics gpu__time_duration.sum --clock-control none -c 600 --csv --log-file captures/launches_r02.csv python bench.py --no-secondary --no-cpu-baseline > /dev/null 2>&1
fi
ls -la captures/*.ncu-rep captures/launches_r02.csv
