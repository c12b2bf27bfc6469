#!/usr/bin/env bash
# compute-sanitizer over every kernel family of libcilantro_b200.so at small sizes (on a GPU machine:
#   bash scripts/sanitize.sh   -> captures/sanitize_{memcheck,racecheck,synccheck}.log
# and a one-line verdict per tool on stdout; tools/sanitize_summary.py turns the logs into a summary).
# memcheck: out-of-bounds / misaligned global, shared and local accesses, leaks of device allocations.
# racecheck: shared-memory hazards between threads of a block (the warp-pooled search queues, the per-warp
#            neighbourhood staging of the robust normals, the barrier-free block reduction, the D-dimensional
#            k-means tiles and the covariance / projection tiles staged between two barriers).
# synccheck: divergent / invalid use of __syncthreads / __syncwarp / *_sync shuffles.
set -u
cd "$(dirname "$0")/.."
mkdir -p captures
SAN=${SAN:-/usr/local/cuda/bin/compute-sanitizer}
rc_all=0
for tool in memcheck racecheck synccheck; do
  extra=""
  [ "$tool" = memcheck ] && extra="--leak-check full"
  log=captures/sanitize_${tool}.log
  SANITIZE_N=${SANITIZE_N:-6000} timeout 1200 "$SAN" --tool "$tool" $extra --error-exitcode 3 --print-limit 400 \
      python tools/sanitize_target.py > "$log" 2>&1
  rc=$?
  summary=$(grep -E "ERROR SUMMARY|RACECHECK SUMMARY|LEAK SUMMARY" "$log" | tr '\n' ' ')
  echo "[$tool] rc=$rc ${summary}"
  grep -q "all checks passed" "$log" || echo "[$tool] the target did not finish"
  [ $rc -ne 0 ] && rc_all=1
done
exit $rc_all
