// Grid-wide deterministic sum reduction used by the accumulation kernels (product code).
#pragma once
#include "cb_internal.hpp"

namespace cb {

// Sums rows r0, r0 + 1, ..., r1 - 1 of a [rows][NV] table into out[NV] with all 256 threads, in a
// fixed order: thread t owns value i = t % IPAD and rows c, c + CH, ... (c = t / IPAD); the CH chunk
// sums of each value are then added in ascending chunk order.
template <int NV>
__device__ __forceinline__ void block_sum_rows(const double* __restrict__ table, unsigned int r0, unsigned int r1,
                                               double* __restrict__ out) {
  constexpr int IPAD = (NV > 16) ? 32 : 16;
  constexpr int CH = kReduceBlock / IPAD;
  __shared__ double red[CH][IPAD];
  const int i = threadIdx.x % IPAD, c = threadIdx.x / IPAD;
  double v = 0;
  if (i < NV)
    for (unsigned int b = r0 + c; b < r1; b += CH) v += __ldcg(table + (size_t)b * NV + i);
  red[c][i] = v;
  __syncthreads();
  if (threadIdx.x < NV) {
    double s = 0;
#pragma unroll
    for (int k = 0; k < CH; k++) s += red[k][threadIdx.x];
    out[threadIdx.x] = s;
  }
  __syncthreads();
}

// warp shuffle -> shared -> one row per block; the last block of each group of kReduceGroup blocks
// folds the group's rows into one group row; the last group folds the group rows into `result`.
// Two levels keep the serial tail short (a single last block summing thousands of rows is a long
// serial tail). Summation order is fixed, so the result does not depend on block
// scheduling. All counters are zero on entry and are left zero.
template <int NV>
__device__ __forceinline__ void grid_reduce(double (&acc)[NV], const ReduceScratch& rs) {
  __shared__ double sm[NV][kReduceBlock / 32];
  __shared__ bool is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < NV; i++) {
    double v = acc[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if (lane == 0) sm[i][warp] = v;
  }
  __syncthreads();
  if (threadIdx.x < NV) {
    double v = 0;
#pragma unroll
    for (int w = 0; w < kReduceBlock / 32; w++) v += sm[threadIdx.x][w];
    rs.partials[(size_t)blockIdx.x * NV + threadIdx.x] = v;
  }
  const unsigned int ngroups = (gridDim.x + kReduceGroup - 1) / kReduceGroup;
  const unsigned int g = blockIdx.x / kReduceGroup;
  const unsigned int g0 = g * kReduceGroup, g1 = min(gridDim.x, g0 + kReduceGroup);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(rs.counters + 1 + g, 1u) == (g1 - g0) - 1);
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  block_sum_rows<NV>(rs.partials, g0, g1, rs.gpartials + (size_t)g * NV);
  if (threadIdx.x == 0) rs.counters[1 + g] = 0;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(rs.counters, 1u) == ngroups - 1);
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  block_sum_rows<NV>(rs.gpartials, 0, ngroups, rs.result);
  if (threadIdx.x == 0) rs.counters[0] = 0;
}

// ---- barrier-free variant -----------------------------------------------------------------------
// Same result and the same fixed summation order, but no warp ever WAITS for another: each warp
// parks its 32-lane sum in its own shared slot and takes a ticket; the warp that arrives last folds
// the block's slots, writes the block row and carries on alone through the group / grid levels.
// Used by the ICP search kernel, whose warps finish at very different times (the barrier version kept
// warps parked at __syncthreads).
template <int NV>
struct AsyncReduceSmem {
  double slot[kReduceBlock / 32][NV];
  unsigned int arrived;
};

// Call once at kernel start (all threads), before any warp can reach grid_reduce_async.
template <int NV>
__device__ __forceinline__ void async_reduce_init(AsyncReduceSmem<NV>& sm) {
  if (threadIdx.x == 0) sm.arrived = 0u;
  __syncthreads();
}

// one warp sums rows r0..r1-1 of a [rows][NV] table; returns the total of value `lane` on lanes < NV.
// NV <= 16: the two half-warps take the even / odd rows (16 loads in flight per lane pair instead of 8 — the fold
// of a group of 64 block rows is a chain of dependent L2 round trips on the tail of every reduction kernel), the two
// half sums are added even + odd. Fixed order in both cases.
template <int NV>
__device__ __forceinline__ double warp_sum_rows(const double* __restrict__ table, unsigned int r0, unsigned int r1,
                                                int lane) {
  double s = 0;
  if constexpr (NV <= 16) {
    const int v = lane & 15, par = lane >> 4;
    if (v < NV) {
      unsigned int b = r0 + par;
      for (; b + 14 < r1; b += 16) {
        double t[8];
#pragma unroll
        for (int u = 0; u < 8; u++) t[u] = __ldcg(table + (size_t)(b + 2 * u) * NV + v);
#pragma unroll
        for (int u = 0; u < 8; u++) s += t[u];
      }
      for (; b < r1; b += 2) s += __ldcg(table + (size_t)b * NV + v);
    }
    const double other = __shfl_xor_sync(0xffffffffu, s, 16);
    s = (par == 0) ? s + other : other + s;  // even rows + odd rows on both halves
  } else {
    if (lane < NV) {
      unsigned int b = r0;
      for (; b + 16 <= r1; b += 16) {
        double t[16];
#pragma unroll
        for (int u = 0; u < 16; u++) t[u] = __ldcg(table + (size_t)(b + u) * NV + lane);
#pragma unroll
        for (int u = 0; u < 16; u++) s += t[u];
      }
      for (; b < r1; ++b) s += __ldcg(table + (size_t)b * NV + lane);
    }
  }
  return s;
}

__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// Fused collective + host notification (struct Exchange, cb_internal.hpp). Called by ONE warp per
// GPU and pass, lane i < NV holding this GPU's total of value i. Returns the cross-rank total.
__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Bit 63 of the host flag / of Exchange-level status words marks a pass whose peer wait timed out.
constexpr unsigned long long kExchangeErrBit = 1ull << 63;

// Steps 1-3 of the fused all-reduce: lane i < NV holds this GPU's total of value i; returns the cross-rank total
// (rows summed in rank order: bit-identical on every rank). The wait for the peers' rows is BOUNDED: if a peer's
// row of this pass has not landed within ex.timeout_ns (a rank that died, never launched its pass, or was
// configured differently), *timed_out is set on every lane and the value returned is meaningless - the caller
// reports the failure (host mailbox flag with kExchangeErrBit / error state of the device loop) instead of
// spinning forever.
template <int NV>
__device__ __forceinline__ double exchange_rows(double s, const Exchange& ex, int lane, bool* timed_out) {
  const int par = (int)(ex.seq & 1ull);
  bool late = false;
  // 1. my row -> every rank's table (remote stores over NVLink), then a release flag per rank
  if (lane < NV)
    for (int p = 0; p < ex.world; ++p) ex.peer_vals[p][(par * ex.world + ex.rank) * kExchangeVals + lane] = s;
  __threadfence_system();
  __syncwarp();
  if (lane < ex.world) st_release_sys(ex.peer_flags[lane] + par * ex.world + ex.rank, ex.seq);
  // 2. wait until every rank's row of THIS pass has landed in my table (lane r watches rank r)
  if (lane < ex.world) {
    const unsigned long long* f = ex.peer_flags[ex.rank] + par * ex.world + lane;
    const unsigned long long t0 = global_timer_ns();
    unsigned int spins = 0;
    while (ld_acquire_sys(f) != ex.seq) {
      if ((++spins & 0xffu) == 0u && ex.timeout_ns != 0ull && global_timer_ns() - t0 > ex.timeout_ns) {
        late = true;
        break;
      }
    }
  }
  late = __any_sync(0xffffffffu, late);
  // 3. identical fixed-order sum on every rank -> bit-identical totals, no broadcast needed
  if (!late && lane < NV) {
    const volatile double* rows = ex.peer_vals[ex.rank] + (size_t)par * ex.world * kExchangeVals;
    s = 0;
    for (int r = 0; r < ex.world; ++r) s += rows[r * kExchangeVals + lane];
  }
  *timed_out = late;
  return s;
}

template <int NV>
__device__ __forceinline__ double exchange_and_publish(double s, const ReduceScratch& rs, int lane) {
  const Exchange& ex = rs.ex;
  if (ex.enabled) {
    bool late = false;
    if (ex.trace && lane == 0) ex.trace[1] = global_timer_ns();  // local reduction done
    if (ex.world > 1) s = exchange_rows<NV>(s, ex, lane, &late);
    if (ex.trace && lane == 0) ex.trace[2] = global_timer_ns();  // peers' rows received and summed
    if (lane < NV) ex.host_vals[lane] = s;
    __threadfence_system();
    __syncwarp();
    if (lane == 0) st_release_sys(ex.host_flag, late ? (ex.seq | kExchangeErrBit) : ex.seq);
    if (ex.trace && lane == 0) ex.trace[3] = global_timer_ns();  // host mailbox flag written
  }
  return s;
}

// Sum NP (16 or 32) per-lane values over the 32 lanes of a warp with a transposing butterfly:
// at each step a lane keeps one half of its values and hands the other half to its partner, so the
// warp spends NP - 1 (+1) shuffles instead of 5 NP. On return v[0] of lane L holds the warp total of
// value L >> 1 (NP = 16, both lanes of a pair hold it) or of value L (NP = 32). Fixed tree order.
template <int NP>
__device__ __forceinline__ double warp_transpose_reduce(double (&v)[NP], int lane) {
  static_assert(NP == 16 || NP == 32, "NP must be 16 or 32");
  int off = 16;
#pragma unroll
  for (int half = NP / 2; half >= 1; half >>= 1) {
    const bool up = (lane & off) != 0;
#pragma unroll
    for (int j = 0; j < half; j++) {
      const double send = up ? v[j] : v[j + half];
      const double keep = up ? v[j + half] : v[j];
      v[j] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
    off >>= 1;
  }
  if (NP == 16) v[0] += __shfl_xor_sync(0xffffffffu, v[0], 1);
  return v[0];
}

// Group / grid levels of the barrier-free reduction, entered by ONE warp per block with lane i < NV holding value i
// of the block's row (a block with nothing to add passes zeros: its row must exist, the folds read every row).
// Returns true on exactly one warp of the grid - the last to arrive - with `tot` = this GPU's total of value `lane`.
template <int NV>
__device__ __forceinline__ bool grid_reduce_rows_tail(double row, const ReduceScratch& rs, int lane, double& tot) {
  unsigned int t = 0;
  if (lane < NV) rs.partials[(size_t)blockIdx.x * NV + lane] = row;
  const unsigned int ngroups = (gridDim.x + kReduceGroup - 1) / kReduceGroup;
  const unsigned int g = blockIdx.x / kReduceGroup;
  const unsigned int g0 = g * kReduceGroup, g1 = min(gridDim.x, g0 + kReduceGroup);
  __threadfence();
  __syncwarp();
  if (lane == 0) t = atomicAdd(rs.counters + 1 + g, 1u);
  t = __shfl_sync(0xffffffffu, t, 0);
  if (t != (g1 - g0) - 1) return false;
  __threadfence();
  {
    const double gs = warp_sum_rows<NV>(rs.partials, g0, g1, lane);
    if (lane < NV) rs.gpartials[(size_t)g * NV + lane] = gs;
  }
  if (lane == 0) rs.counters[1 + g] = 0;
  __threadfence();
  __syncwarp();
  if (lane == 0) t = atomicAdd(rs.counters, 1u);
  t = __shfl_sync(0xffffffffu, t, 0);
  if (t != ngroups - 1) return false;
  __threadfence();
  // the last warp of the grid: this GPU's totals
  tot = warp_sum_rows<NV>(rs.gpartials, 0, ngroups, lane);
  if (lane == 0) rs.counters[0] = 0;
  return true;
}

// The warp's sums of acc[] -> its slot of the block row: stored (kAdd = false) or added to what the warp parked there
// before (kAdd = true; the slot must then have been zeroed by the warp). Fixed order.
// kAdd is for callers that fold acc[] inside a loop and go on accumulating: it reduces value by value, because ptxas
// turns the transposing butterfly's selects into indexed local-memory loads, and inside a loop that kept a local copy
// of acc[] written on every accumulation.
template <int NV, bool kAdd>
__device__ __forceinline__ void warp_sum_to_slot(double (&acc)[NV], AsyncReduceSmem<NV>& sm) {
  static_assert(NV <= 32, "one lane per value");
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if constexpr (NV == 16 && !kAdd) {
    const double t16 = warp_transpose_reduce<16>(acc, lane);
    if ((lane & 1) == 0) sm.slot[warp][lane >> 1] = t16;
  } else {
#pragma unroll
    for (int i = 0; i < NV; i++) {
      double v = acc[i];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
      if (lane == 0) sm.slot[warp][i] = kAdd ? sm.slot[warp][i] + v : v;
    }
  }
  __syncwarp();
}

// Block level once every warp of the block has filled its slot (warp_sum_to_slot): returns true on exactly one warp
// of the block - the last to arrive - with `row` = the block's total of value `lane` (lane < NV; zero on the other
// lanes). Fixed order.
template <int NV>
__device__ __forceinline__ bool block_row_from_slots(AsyncReduceSmem<NV>& sm, double& row) {
  const int lane = threadIdx.x & 31;
  constexpr int kWarps = kReduceBlock / 32;
  unsigned int t = 0;
  if (lane == 0) {
    __threadfence_block();
    t = atomicAdd(&sm.arrived, 1u);
  }
  t = __shfl_sync(0xffffffffu, t, 0);
  if (t != kWarps - 1) return false;
  __threadfence_block();
  row = 0;
  if (lane < NV) {
#pragma unroll
    for (int w = 0; w < kWarps; w++) row += ((volatile double*)sm.slot[w])[lane];
  }
  return true;
}

// warp -> block -> group -> grid without a barrier (the last warp of the grid carries on alone) -> (optional) fused
// all-reduce over NVLink peer memory -> device result + mapped host mailbox
template <int NV>
__device__ __forceinline__ void grid_reduce_async(double (&acc)[NV], const ReduceScratch& rs, AsyncReduceSmem<NV>& sm) {
  const int lane = threadIdx.x & 31;
  warp_sum_to_slot<NV, false>(acc, sm);
  double row, tot = 0;
  if (!block_row_from_slots<NV>(sm, row)) return;
  if (!grid_reduce_rows_tail<NV>(row, rs, lane, tot)) return;
  tot = exchange_and_publish<NV>(tot, rs, lane);
  if (lane < NV) rs.result[lane] = tot;
}

// ---- one block folds a whole grid's rows ------------------------------------------------------------------------
// Sums rows 0 .. rows-1 of a [rows][NV] table (one row per block of the kernel that ran before; launched after it,
// so no ticket is needed) with the kReduceBlock threads of ONE block, into out[NV] (shared memory). The result is
// bit-identical to the two ticketed levels of grid_reduce_rows_tail: groups of kReduceGroup consecutive rows, each
// summed by warp_sum_rows' rule (NV <= 16: even and odd rows separately in ascending order, then even + odd; else
// ascending), then the group rows by the same rule.
// Thread work item: (group, parity, pair of adjacent values); its rows are loaded 16 B at a time, kFoldBatch of them in
// flight, and added in ascending order. A round covers the groups that one item per thread reaches; the round's
// group rows go through shared memory to the threads that carry the grid-level sums, in ascending group order.
template <int NV>
__device__ __forceinline__ void block_fold_rows(const double* __restrict__ table, unsigned int rows, double* out) {
  static_assert(NV % 2 == 0, "values are loaded in pairs");
  constexpr int kPar = (NV <= 16) ? 2 : 1;                 // parities summed apart (warp_sum_rows)
  constexpr int kPairs = NV / 2;
  constexpr int kItemsPerGroup = kPar * kPairs;
  constexpr int kRoundGroups = kReduceBlock / kItemsPerGroup;  // even: group parity = parity within the round
  constexpr int kFoldBatch = 32;
  static_assert(kRoundGroups % 2 == 0, "group parity");
  __shared__ double part[kRoundGroups][kPar][NV];
  __shared__ double grid_par[kPar][NV];
  const unsigned int tid = threadIdx.x;
  const unsigned int ngroups = (rows + kReduceGroup - 1) / kReduceGroup;
  const unsigned int gl = tid / kItemsPerGroup, par = (tid % kItemsPerGroup) / kPairs, v = 2 * (tid % kPairs);
  double acc = 0;  // grid level: thread tid < kPar * NV sums value tid % NV over the groups of parity tid / NV
  for (unsigned int g0 = 0; g0 < ngroups; g0 += kRoundGroups) {
    const unsigned int g = g0 + gl;
    if (gl < kRoundGroups && g < ngroups) {
      const unsigned int r1 = min(rows, (g + 1) * kReduceGroup);
      double sx = 0, sy = 0;
      for (unsigned int r = g * kReduceGroup + par; r < r1; r += kFoldBatch * kPar) {
        double2 t[kFoldBatch];
#pragma unroll
        for (int u = 0; u < kFoldBatch; u++) {
          const unsigned int b = r + u * kPar;
          if (b < r1) t[u] = __ldcg(reinterpret_cast<const double2*>(table + (size_t)b * NV + v));
        }
#pragma unroll
        for (int u = 0; u < kFoldBatch; u++)
          if (r + u * kPar < r1) {
            sx += t[u].x;
            sy += t[u].y;
          }
      }
      part[gl][par][v] = sx;
      part[gl][par][v + 1] = sy;
    }
    __syncthreads();
    if (tid < kPar * NV) {
      const unsigned int p = tid / NV, i = tid % NV;
      for (unsigned int k = p; k < kRoundGroups && g0 + k < ngroups; k += kPar)
        acc += (kPar == 2) ? part[k][0][i] + part[k][kPar - 1][i] : part[k][0][i];
    }
    __syncthreads();
  }
  if (tid < kPar * NV) grid_par[tid / NV][tid % NV] = acc;
  __syncthreads();
  if (tid < NV) out[tid] = (kPar == 2) ? grid_par[0][tid] + grid_par[kPar - 1][tid] : grid_par[0][tid];
  __syncthreads();
}

}  // namespace cb
