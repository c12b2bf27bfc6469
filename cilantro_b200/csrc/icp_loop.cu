// Device-resident rigid ICP loop (product code, sm_90a).
//
// IterativeClosestPointBase::estimate() (registration/icp_base.hpp:68-87) for the default correspondence engine:
// ONE kernel per ICP iteration and NO host round trip between iterations. The kernel of iteration k
//   1. reads the current estimate T_k from device memory (LoopState),
//   2. finds every source point's correspondence under T_k (below),
//   3. accumulates the estimator's moments and reduces them warp -> block -> grid in a fixed order,
//   4. in the ONE warp that finishes the grid reduction: all-reduces the 16 / 28 totals with the peer ranks over
//      NVLink peer memory (reduce.cuh, bounded wait), then solves on the device — Kabsch / one Gauss-Newton step,
//      rotation() re-orthonormalisation, compose, update norm, convergence test (solve_core.hpp; the same code the
//      host loop runs) — and writes T_{k+1} back to LoopState.
// The host enqueues the launches back to back and reads LoopState once per batch; launches after convergence
// return at once. With several ranks every rank solves the same totals redundantly -> bit-identical transforms.
//
// Correspondences WITHOUT a search (exact). Every search also returns an EXCLUSION bound: a radius r such that
// every reference point other than the match is at least r away from the query (warp_search_wide.cuh). The next
// iteration moves the query by delta = |T_{k+1} s - T_k s|, so every other point is still at least r - delta away
// (triangle inequality); if the cached match's distance under T_{k+1} — evaluated with the contract arithmetic,
// i.e. the very number the search would compute for it — is below that, the match is provably still the unique
// nearest neighbour and its (index, d2) is what the full search would return, bit for bit. Only the queries
// that fail the test are searched again, inside the same pass: each warp queues the ones it flagged, so the search
// runs on dense warps. All bounds are rounded conservatively (directed rounding + 2^-18 relative margins, far above the
// 6-ulp error of the fp32 distance evaluation); an exact tie can never pass the strict test.
// As ICP converges the per-iteration motion shrinks geometrically and almost every query takes the cached path:
// the iteration becomes one streaming pass (16 B query + 8 B cache + one 16 B gather per source point).
#include "cache_rule.hpp"
#include "icp_accumulate.cuh"
#include "icp_kernels.cuh"
#include "icp_object.hpp"
#include "reduce.cuh"
#include "solve_core.hpp"
#include "solve_warp.cuh"
#include "warp_search_wide.cuh"
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

namespace cb {

namespace {

constexpr int kBlock = kReduceBlock;

struct LoopArgs {
  GridView dst;
  const float4* src_pts;  // cell-sorted query cloud; .w = original index bits
  const float4* src_nrm;  // same order, or nullptr (symmetric metric when set)
  uint32_t n_src;
  float max_d2, w_pt, w_pl, tol;
  int wk_pt, wk_pl;    // cb_weight_kind of the correspondence weight evaluators (combined metric)
  float wc_pt, wc_pl;  // RBF coefficients
  float dm[3];        // dst_mean_
  float src_mean[3];  // src_mean_ (the kernel applies the current transform)
  int has_pt, has_pl;  // combined metric: which terms are on
  int bail;            // plane terms wanted but dst has no normals -> identity update (transform_estimation.hpp:269-272)
  int* cache_pos;      // per sorted query: sorted dst position of its match (-1 none)
  float* cache_r;      // per sorted query: every OTHER dst point is at least this far away (<= 0: unknown)
  float slack_first, slack_min, slack_max;  // widening of the search beyond the nearest distance (warp_search_wide.cuh)
  LoopState* st;
  ReduceScratch rs;
  int trace;  // CB_LOOP_TRACE: fill LoopState::trace
};

// per-block copy of the loop state; also the `Args` of accumulate_pair (T, dm, sm, w_pt, w_pl)
struct BlockCtx {
  Rigid T, Tp;
  float dm[3], sm[3];
  float w_pt, w_pl;
  int wk_pt, wk_pl;
  float wc_pt, wc_pl;
  int have_prev, done;
};

__device__ __forceinline__ Rigid rigid_from_t12_dev(const float* T12) {
  Rigid r;
#pragma unroll
  for (int i = 0; i < 3; i++) {
#pragma unroll
    for (int j = 0; j < 3; j++) r.r[i * 3 + j] = __ldcg(T12 + i * 4 + j);
    r.t[i] = __ldcg(T12 + i * 4 + 3);
  }
  return r;
}

// The serial epilogue of an iteration (one thread): totals -> update -> new state. It runs in a kernel of its own
// (icp_finish_kernel, one warp): inside the search kernel its temporaries were spilled at that kernel's register
// budget, and a spilled word of ONE thread lives in its own 128-byte line of local memory - after a 10 M-point pass
// every one of them was a cold DRAM miss (in a %globaltimer trace the solve took many times its arithmetic).
template <int MODE>
__device__ __forceinline__ void loop_solve(const LoopArgs* ap, const BlockCtx* cxp, const double* s, int late,
                                        unsigned long long seq) {
  const LoopArgs& a = *ap;
  const BlockCtx& cx = *cxp;
  LoopState* st = a.st;
  if (late) {  // a peer's row never arrived (reduce.cuh, exchange_rows)
    st->error = CB_ERR_NCCL;
    st->done = 2;
    __threadfence();
    return;
  }
  float T[12], Titer[12], Tn[12];
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) T[i * 4 + j] = cx.T.r[i * 3 + j];
    T[i * 4 + 3] = cx.T.t[i];
  }
  if (MODE == kModeP2PCentered) {
    sc::kabsch_from_moments(s, cx.dm, cx.sm, Titer);  // transform_estimation.hpp:12-48
  } else {
    // estimateTransformCombinedMetric, max_iter = 1 (transform_estimation.hpp:238-367 / :608-739)
    const bool has_terms = s[0] > 0.0 && (a.has_pt || a.has_pl);
    if (!has_terms || a.bail) {
      sc::t34_identity(Titer);
    } else {
      float I[12], dn = 0.f;
      sc::t34_identity(I);
      sc::gauss_newton_apply(s + kCombinedValues, I, Titer, &dn);  // d_theta solved by the whole warp (solve6_warp)
      sc::uncenter(Titer, cx.dm, cx.sm);
    }
  }
  sc::reorthonormalize(Titer);                  // icp_single_transform_combined_metric.hpp:207-211
  sc::compose(Titer, T, Tn);                    // :213
  const float delta = sc::update_norm(Titer);   // :214-216
  for (int i = 0; i < 12; i++) {
    st->T_prev[i] = T[i];
    st->T[i] = Tn[i];
    st->Titer[i] = Titer[i];
  }
  for (int i = 0; i < 28; i++) st->sums[i] = (i < (MODE == kModeP2PCentered ? kP2PValues : kCombinedValues)) ? s[i] : 0.0;
  st->last_delta = delta;
  st->iters = st->iters + 1;
  st->n_corr = s[0];
  st->have_prev = 1;
  st->xseq = seq;
  st->searched_last = st->searched_cur;
  st->searched_cur = 0ull;
  if (delta < a.tol) st->done = 1;  // icp_base.hpp:83
  if (a.trace) {
    st->trace[(st->iters - 1) & 63][3] = global_timer_ns();
    st->trace[st->iters & 63][5] = 0ull;  // the next iteration's kernels take the maximum over their warps
  }
  __threadfence();
}

// One lane-dense warp search (query i on every lane with act set) and cache update. Returns the searching lane's
// pair: query index i, transformed query q, match position pos (-1 none / inactive lane).
struct ChunkPair {
  uint32_t i;
  int pos;
  float qx, qy, qz;
  float d2;  // the match's squared distance (correspondence value)
};

// Lanes per queued region in the wide search's pooled scan (warp_search_wide.cuh). The cold search keeps one lane per
// region. The cached pass's search uses pairs of lanes: its region scan then needs fewer live registers, and the
// pass's streaming loop, which holds the call site of search_chunk_far, spills less (DESIGN §4.2).
constexpr unsigned int kColdGroup = 1, kWarmGroup = 2;
// kCold: nothing cached yet (no warm seed, first-iteration slack). Otherwise the query failed the exclusion test:
// its cached match seeds the search and its last motion sets the slack.
template <bool kCold>
__device__ __forceinline__ ChunkPair search_chunk_body(const LoopArgs& a, const BlockCtx& cx, WideSearchSmem* wsm,
                                                       bool act, uint32_t i) {
  ChunkPair cp;
  cp.i = i;
  cp.pos = -1;
  cp.qx = cp.qy = cp.qz = 0.f;
  cp.d2 = 0.f;
  float slack = a.slack_first;
  int sd = -1;
  if (act) {
    const float4 s = __ldg(a.src_pts + cp.i);
    rule::transform_point(cx.T, s.x, s.y, s.z, cp.qx, cp.qy, cp.qz);
    if (!kCold) {
      float ox, oy, oz;
      rule::transform_point(cx.Tp, s.x, s.y, s.z, ox, oy, oz);
      const float ex = __fsub_rn(cp.qx, ox), ey = __fsub_rn(cp.qy, oy), ez = __fsub_rn(cp.qz, oz);
      const float dl = __fsqrt_ru(__fmaf_ru(ez, ez, __fmaf_ru(ey, ey, __fmul_ru(ex, ex))));
      // the next step is expected to be about half of this one, and a hit needs r - (motion) > d: widen by 2 x
      slack = fminf(fmaxf(__fmul_rn(2.f, dl), a.slack_min), a.slack_max);
      sd = a.cache_pos[cp.i];
    }
  }
  const WideBest wb = warp_grid_nearest_wide<kCold ? kColdGroup : kWarmGroup>(a.dst, *wsm, act, cp.qx, cp.qy, cp.qz, a.max_d2, sd, slack);
  if (act) {
    cp.pos = (wb.idx >= 0 && wb.d2 < a.max_d2) ? wb.pos : -1;
    cp.d2 = wb.d2;
    a.cache_pos[cp.i] = cp.pos;
    a.cache_r[cp.i] = rule::cache_radius(wb.D2);
  }
  return cp;
}

// Out-of-line search of the cached pass: called from inside its tile loop, where the streaming registers and the
// moment accumulators are live. Inlined there, the search's loop-invariant parameter loads were hoisted into
// registers and the streaming loop spilled; behind the call only the call site saves and restores registers, once per
// warp search.
__device__ __noinline__ void search_chunk_far(const LoopArgs* ap, const BlockCtx* cxp, WideSearchSmem* wsm, bool act,
                                              uint32_t i, ChunkPair* out) {
  *out = search_chunk_body<false>(*ap, *cxp, wsm, act, i);
}

// Programmatic dependent launch (sm_90+): a kernel launched with the programmatic-stream-serialization attribute may
// be scheduled while its predecessor in the stream is still running; it must execute pdl_wait() before it touches
// anything the predecessor (or, transitively, earlier kernels: the predecessor passed its own pdl_wait first) wrote.
// The predecessor allows that early scheduling with pdl_launch_dependents(). Used between the two kernels of an
// iteration so that the launch latency of the next kernel overlaps the tail of the previous one.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// thread 0 of a block: LoopState -> shared BlockCtx
__device__ __forceinline__ void load_block_ctx(const LoopArgs& a, BlockCtx& cx) {
  cx.done = __ldcg(&a.st->done);
  cx.have_prev = __ldcg(&a.st->have_prev);
  cx.T = rigid_from_t12_dev(a.st->T);
  cx.Tp = rigid_from_t12_dev(a.st->T_prev);
  float smx, smy, smz;
  rule::transform_point(cx.T, a.src_mean[0], a.src_mean[1], a.src_mean[2], smx, smy, smz);  // transform_ * src_mean_
  cx.sm[0] = smx; cx.sm[1] = smy; cx.sm[2] = smz;
  cx.dm[0] = a.dm[0]; cx.dm[1] = a.dm[1]; cx.dm[2] = a.dm[2];
  cx.w_pt = a.w_pt;
  cx.w_pl = a.w_pl;
  cx.wk_pt = a.wk_pt;
  cx.wk_pl = a.wk_pl;
  cx.wc_pt = a.wc_pt;
  cx.wc_pl = a.wc_pl;
}

// ---- kernel 1 of a warm iteration: the cached pass and the search of what it could not decide ---------------------
// Elementwise over the source cloud: per query 16 B (point) + 8 B (cache) streamed and one 16 B gather of the cached
// match (+ 16 B normal for the plane term). Queries that pass the exclusion test accumulate their pair at once. The
// others are searched by the warp that flagged them: after each 32-query slot the warp's ballot appends the flagged
// query indices, in ascending order, to a warp-private queue; as soon as 32 are queued the warp searches them
// lane-dense (search_chunk_far: same slack rule, warm seed and cache update as the cold search), and at the end of its
// tiles it searches what is left. Only __syncwarp is involved, so a searching warp holds up no other warp of its
// block, and the searching lane adds its pair to the same accumulators.
// PERSISTENT: the grid is a whole number of resident blocks per SM, a block walks the tiles blockIdx.x, + gridDim.x,
// ... (static round-robin: every tile costs the same, and the assignment — hence, with the fixed queue order, the
// summation order — is fixed), the next tiles' loads are in flight while the current tile is evaluated, and the
// moments are reduced ONCE per block (a per-tile reduction cost as much as the tile itself). The block rows go through
// one deterministic grid reduction per iteration into rs.result, read by the finish kernel.
// The loads are not staged in registers: a register-staged version needed 128 registers -> 2 blocks/SM, few warp
// slots occupied, long-scoreboard stalls on top - each thread can only keep the loads in flight that it has registers
// for. Here every thread runs a private three-deep pipeline of cp.async copies into shared memory (LDGSTS: no
// destination register, no scoreboard slot):
//   stage A (tile k+2)  the streamed arrays: its queries' point (16 B), exclusion radius (4 B), cached match (4 B)
//   stage B (tile k+1)  the gathers, once A has landed: the matched destination point (+ normal for the plane term)
//   stage C (tile k)    evaluation from shared memory
// Each thread only ever reads what it copied itself, so cp.async.wait_group is all the synchronisation there is -
// no block barrier inside the tile loop.
// Shared memory per block: the pipeline (three A buffers, two B buffers) and one WideSearchSmem per warp (27.6 KB,
// the queue included), 1 KB of reduction slots and state.
//   p2p: 256-query tiles (one query per thread): 26 KB of pipeline, 56 KB per block -> 4 blocks per SM in the 228 KB
//        of an H100 SM, 64 registers. (512-query tiles would need 82 KB per block: 2 blocks per SM.)
//   combined: 512-query tiles: 68 KB of pipeline, 98 KB per block -> 2 blocks per SM, 128 registers. At 3 blocks
//        (80 registers, 256-query tiles) the exclusion test and the 28 accumulators spilled on every query, and with
//        3 x 65 KB of shared memory the L1 left for those spills was too small: the 10 M pass ran 3x slower.
// Both keep 1024 queries per SM in flight in the pipeline.
__host__ __device__ constexpr int pipe_qpt(bool normals) { return normals ? 2 : 1; }
__host__ __device__ constexpr int pipe_min_blocks(bool normals) { return normals ? 2 : 4; }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async_16_cg(void* dst_smem, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_16_ca(void* dst_smem, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_4(void* dst_smem, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

template <bool kNormals>
struct PipeSmem {
  static constexpr int kT = pipe_qpt(kNormals) * kBlock;  // queries per tile
  float4 src[3][kT];
  float r[3][kT];
  int seed[3][kT];
  float4 pt[2][kT];
  float4 nr[kNormals ? 2 : 1][kNormals ? kT : 1];
};

template <int MODE>
__global__ void __launch_bounds__(kBlock, pipe_min_blocks(MODE == kModeCombined)) icp_cached_pipe_kernel(const __grid_constant__ LoopArgs a) {
  constexpr int NV = (MODE == kModeP2PCentered) ? kP2PValues : kCombinedValues;
  constexpr bool kNormals = (MODE == kModeCombined);
  constexpr int kQpt = pipe_qpt(kNormals), kTile = kQpt * kBlock;
  extern __shared__ __align__(16) unsigned char pipe_raw[];
  PipeSmem<kNormals>& ps = *reinterpret_cast<PipeSmem<kNormals>*>(pipe_raw);
  __shared__ BlockCtx cx;
  __shared__ AsyncReduceSmem<NV> rsm;
  __shared__ WideSearchSmem wsm[kBlock / 32];
  const unsigned int tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  // per warp: flagged query indices waiting for a search, ascending. The queue lives in the warp's search buffer: it
  // is only filled between searches, and each lane reads its entry before the search overwrites the buffer. (A queue
  // of its own, 1 KB per block, would leave the p2p pass 176 B short of 4 blocks per SM.)
  uint32_t* wq = wsm[warp].sec;
  const uint32_t ntiles = (a.n_src + kTile - 1) / kTile;
  const bool want_nrm = kNormals && a.has_pl != 0;

  // stage A of tile `tile` into buffer `buf`: nothing here depends on the loop state
  auto stage_a = [&](uint32_t tile, int buf) {
    if (tile < ntiles) {
#pragma unroll
      for (int k = 0; k < kQpt; k++) {
        const uint32_t slot = k * kBlock + tid, i = tile * kTile + slot;
        if (i < a.n_src) {
          cp_async_16_cg(&ps.src[buf][slot], a.src_pts + i);
          cp_async_4(&ps.r[buf][slot], a.cache_r + i);
          cp_async_4(&ps.seed[buf][slot], a.cache_pos + i);
        }
      }
    }
    cp_async_commit();
  };
  // stage B: the gathers of tile `tile` (its stage A has landed in abuf) into bbuf
  auto stage_b = [&](uint32_t tile, int abuf, int bbuf) {
    if (tile < ntiles) {
#pragma unroll
      for (int k = 0; k < kQpt; k++) {
        const uint32_t slot = k * kBlock + tid, i = tile * kTile + slot;
        if (i < a.n_src) {
          const int sd = ps.seed[abuf][slot];
          if (sd >= 0 && ps.r[abuf][slot] > 0.f) {
            cp_async_16_ca(&ps.pt[bbuf][slot], a.dst.pts + sd);
            if (kNormals && want_nrm) cp_async_16_ca(&ps.nr[bbuf][slot], a.dst.nrm + sd);
          }
        }
      }
    }
    cp_async_commit();
  };

  const uint32_t t0 = blockIdx.x, stride = gridDim.x;
  // The dependency wait comes BEFORE the first copies: the cache arrays are rewritten every iteration, their 4-byte
  // copies go through L1 (cp.async.ca), and only accesses after griddepcontrol.wait are guaranteed to see the previous
  // kernels' writes. What programmatic launch buys here: the blocks are resident when the finish kernel ends, and the
  // one-warp finish kernel of this iteration, released at once, is resident and waiting when this grid drains.
  pdl_wait();
  pdl_launch_dependents();
  stage_a(t0, 0);           // group: A(0)
  stage_a(t0 + stride, 1);  // group: A(1)
  if (tid == 0) {
    rsm.arrived = 0u;
    load_block_ctx(a, cx);
  }
  __syncthreads();
  if (cx.done) {
    cp_async_wait<0>();
    return;
  }
  if (a.trace && blockIdx.x == 0 && tid == 0) {
    const int slot = __ldcg(&a.st->iters) & 63;
    a.st->trace[slot][0] = global_timer_ns();
    a.st->trace[slot][4] = 0ull;
  }
  cp_async_wait<1>();   // A(0) has landed
  stage_b(t0, 0, 0);    // group: B(0)
  double acc[NV];
#pragma unroll
  for (int v = 0; v < NV; v++) acc[v] = 0.0;
  // the warp's row of the block reduction: what the warp folded before each search (and, at the end, the rest)
  if (lane < NV) rsm.slot[warp][lane] = 0.0;
  __syncwarp();  // (lane 0 adds to the whole row)
  // The warp searches the queries queued in wq[0, n) on lanes < n; the searching lane accumulates its pair. The
  // accumulators are folded into the warp's row first and restart from zero, so that no register of the streaming
  // loop is live across the search call (held there, all of acc[] was kept in local memory for the whole loop).
  unsigned int queued = 0, searched = 0;  // warp-uniform
  auto search_queued = [&](unsigned int n) {
    __syncwarp();
    warp_sum_to_slot<NV, true>(acc, rsm);
#pragma unroll
    for (int v = 0; v < NV; v++) acc[v] = 0.0;
    const bool act = lane < n;
    ChunkPair cp;
    search_chunk_far(&a, &cx, &wsm[warp], act, act ? wq[lane] : 0u, &cp);
    if (cp.pos >= 0) {
      const float4 dp = __ldg(a.dst.pts + cp.pos);
      accumulate_pair<MODE, true>(
          acc, cx, a.has_pt != 0, a.has_pl != 0, dp, cp.qx, cp.qy, cp.qz, a.src_nrm != nullptr,
          [&] { return __ldg(a.dst.nrm + cp.pos); }, [&] { return __ldg(a.src_nrm + cp.i); }, cp.d2);
    }
    searched += n;
    __syncwarp();  // every lane has read its entry before the queue is refilled
  };
  // iteration n evaluates tile t0 + n*stride; on entry the committed groups are ... A(n+1), B(n)
  int abuf = 0, bbuf = 0;
#pragma unroll 1
  for (uint32_t tile = t0; tile < ntiles; tile += stride) {
    const int abuf1 = (abuf == 2) ? 0 : abuf + 1, abuf2 = (abuf1 == 2) ? 0 : abuf1 + 1;
    stage_a(tile + 2 * stride, abuf2);             // group: A(n+2)
    cp_async_wait<2>();                            // pending at most {B(n), A(n+2)}: A(n+1) has landed
    stage_b(tile + stride, abuf1, bbuf ^ 1);       // group: B(n+1)
    cp_async_wait<2>();                            // pending at most {A(n+2), B(n+1)}: B(n) has landed
    const uint32_t base = tile * kTile;
#pragma unroll
    for (int k = 0; k < kQpt; k++) {
      const uint32_t slot = k * kBlock + tid, i = base + slot;
      const bool active = i < a.n_src;
      bool miss = active;
      if (active) {
        const float rc = ps.r[abuf][slot];
        const int sd = ps.seed[abuf][slot];
        if (rc > 0.f) {
          const float4 sc = ps.src[abuf][slot];
          // the exclusion test (cache_rule.hpp): hit -> the cached match is this iteration's exact search result
          rule::Verdict v;
          float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
          rule::cached_match_test(cx.T, cx.Tp, sc.x, sc.y, sc.z, rc, sd, a.max_d2, [&] { return ps.pt[bbuf][slot]; }, p, v);
          miss = v.miss;
          if (!miss) a.cache_r[i] = v.r2;
          if (v.pair) {
            accumulate_pair<MODE, true>(
                acc, cx, a.has_pt != 0, a.has_pl != 0, p, v.qx, v.qy, v.qz, a.src_nrm != nullptr,
                [&] { return kNormals ? ps.nr[kNormals ? bbuf : 0][kNormals ? slot : 0] : make_float4(0.f, 0.f, 0.f, 0.f); },
                [&] { return __ldg(a.src_nrm + i); }, v.d2);
          }
        }
      }
      // flagged queries -> the warp's queue; the ones that do not fit wait in their lane's register (i) until the
      // 32 queued ones have been searched
      const unsigned int mm = __ballot_sync(0xffffffffu, miss);
      const unsigned int at = queued + __popc(mm & ((1u << lane) - 1u));
      if (miss && at < 32u) wq[at] = i;
      queued += __popc(mm);
      if (queued >= 32u) {
        search_queued(32u);
        queued -= 32u;
        if (miss && at >= 32u) wq[at - 32u] = i;
      }
    }
    abuf = abuf1;
    bbuf ^= 1;
  }
  cp_async_wait<0>();
  if (queued > 0u) search_queued(queued);
  if (lane == 0 && searched > 0u) {
    atomicAdd(&a.st->searched_cur, (unsigned long long)searched);
    if (a.trace) atomicAdd(&a.st->trace[__ldcg(&a.st->iters) & 63][4], (unsigned long long)searched);
  }
  if (a.trace && lane == 0) atomicMax(&a.st->trace[__ldcg(&a.st->iters) & 63][5], global_timer_ns());
  warp_sum_to_slot<NV, true>(acc, rsm);
  double tot = 0;
  if (!grid_reduce_slots_tail<NV>(a.rs, rsm, tot)) return;
  // the last warp of the grid hands this GPU's totals to icp_finish_kernel
  if (lane < NV) a.rs.result[lane] = tot;
  if (a.trace && lane == 0) a.st->trace[__ldcg(&a.st->iters) & 63][1] = global_timer_ns();
}

constexpr int kSearchMinBlocks = 4;  // resident blocks per SM the search kernel's register budget is set for

// ---- the cold iteration (the first of a call: nothing cached yet): search, then the finish kernel -----------------
// Every query is searched, one 256-query chunk per block, lane-dense; the searching thread accumulates its pair and
// the last warp of the grid hands this GPU's totals to icp_finish_kernel.
template <int MODE>
__global__ void __launch_bounds__(kBlock, kSearchMinBlocks) icp_search_kernel(const __grid_constant__ LoopArgs a) {
  constexpr int NV = (MODE == kModeP2PCentered) ? kP2PValues : kCombinedValues;
  __shared__ BlockCtx cx;
  __shared__ WideSearchSmem wsm[kBlock / 32];
  __shared__ AsyncReduceSmem<NV> rsm;

  const unsigned int tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const uint32_t base = blockIdx.x * kBlock;
  pdl_wait();               // the state of the previous finish kernel
  pdl_launch_dependents();  // the one-warp finish kernel may be scheduled now and wait for this grid to drain
  if (tid == 0) {
    rsm.arrived = 0u;
    load_block_ctx(a, cx);
  }
  __syncthreads();
  if (cx.done) return;  // converged (or failed) in an earlier launch of this batch
  const int trace_slot = a.trace ? (__ldcg(&a.st->iters) & 63) : 0;
  if (a.trace && blockIdx.x == 0 && tid == 0) {
    a.st->trace[trace_slot][0] = global_timer_ns();
    a.st->trace[trace_slot][4] = 0ull;
  }
  const unsigned int total = (base < a.n_src) ? min((uint32_t)kBlock, a.n_src - base) : 0u;
  if (tid == 0 && total > 0) {
    atomicAdd(&a.st->searched_cur, (unsigned long long)total);
    if (a.trace) atomicAdd(&a.st->trace[trace_slot][4], (unsigned long long)total);
  }
  double acc[NV];
#pragma unroll
  for (int v = 0; v < NV; v++) acc[v] = 0.0;
  if ((tid & ~31u) < total) {
    const ChunkPair cp = search_chunk_body<true>(a, cx, &wsm[warp], tid < total, base + tid);
    if (cp.pos >= 0) {
      const float4 dp = __ldg(a.dst.pts + cp.pos);
      accumulate_pair<MODE, true>(
          acc, cx, a.has_pt != 0, a.has_pl != 0, dp, cp.qx, cp.qy, cp.qz, a.src_nrm != nullptr,
          [&] { return __ldg(a.dst.nrm + cp.pos); }, [&] { return __ldg(a.src_nrm + cp.i); }, cp.d2);
    }
  }
  if (a.trace && lane == 0) atomicMax(&a.st->trace[trace_slot][5], global_timer_ns());
  double tot = 0;
  if (!grid_reduce_async_tail<NV>(acc, a.rs, rsm, tot)) return;
  if (lane < NV) a.rs.result[lane] = tot;
  if (a.trace && lane == 0) a.st->trace[trace_slot][1] = global_timer_ns();
}

// ---- kernel 3 of an iteration: exchange + solve (one warp) -------------------------------------------------------------
// This GPU's totals -> all-reduce with the peer ranks over NVLink peer memory (reduce.cuh, bounded wait; every rank
// sums the rows in rank order -> bit-identical totals) -> Kabsch / Gauss-Newton step, rotation(), compose,
// convergence test -> LoopState for the next iteration's kernels.
template <int MODE>
__global__ void __launch_bounds__(32, 1) icp_finish_kernel(const __grid_constant__ LoopArgs a) {
  constexpr int NV = (MODE == kModeP2PCentered) ? kP2PValues : kCombinedValues;
  __shared__ BlockCtx cx;
  __shared__ double sbuf[kCombinedValues + 8];
  static_assert(NV + 2 <= kExchangeVals, "row of the fused exchange");
  const unsigned int lane = threadIdx.x;
  pdl_wait();               // this GPU's totals (cached pass or cold search kernel), the state of the previous iteration
  pdl_launch_dependents();  // the next iteration's cached pass may start streaming
  if (lane == 0) load_block_ctx(a, cx);
  __syncwarp();
  if (cx.done) return;
  const int trace_slot = a.trace ? (__ldcg(&a.st->iters) & 63) : 0;
  // lanes < NV: the moments; lane NV: queries this rank searched in this iteration; lane NV + 1: its source points
  // (both ride along so that every rank sees the same global search share: the hand-over decision of the host)
  double tot = (lane < NV) ? __ldcg(a.rs.result + lane) : 0.0;
  if (lane == NV) tot = (double)__ldcg(&a.st->searched_cur);
  if (lane == NV + 1) tot = (double)a.n_src;
  bool late = false;
  const unsigned long long seq = __ldcg(&a.st->xseq) + 1ull;
  if (a.rs.ex.enabled && a.rs.ex.world > 1) {
    Exchange ex = a.rs.ex;
    ex.seq = seq;  // executed passes are numbered on the device: launches skipped after convergence take no number
    tot = exchange_rows<NV + 2>(tot, ex, (int)lane, &late);
  }
  if (lane == NV) a.st->searched_all = tot;
  if (lane == NV + 1) a.st->queries_all = tot;
  if (a.trace && lane == 0) a.st->trace[trace_slot][2] = global_timer_ns();
  if (lane < NV) sbuf[lane] = tot;
  __syncwarp();
  if constexpr (MODE == kModeCombined) {
    // d_theta = AtA^-1 Atb with the augmented matrix spread over the warp, parked behind the totals
    double x[6];
    solve6_warp(sbuf, (int)lane, x);
    if (lane == 0)
#pragma unroll
      for (int i = 0; i < 6; i++) sbuf[kCombinedValues + i] = x[i];
    __syncwarp();
  }
  if (lane == 0) loop_solve<MODE>(&a, &cx, sbuf, late ? 1 : 0, seq);
}

}  // namespace

// widening of a search beyond the nearest distance, in cell edges of the destination grid: first iteration
// (no motion known yet), floor and cap of 2 x (the query's last motion)
constexpr float kSlackFirst = 0.20f, kSlackMin = 0.02f, kSlackMax = 0.30f;
constexpr int kBatch = 16;  // iterations per batch after the first one (the host reads LoopState once per batch)
// The first batch is short: by its end a converging run searches a fraction of a percent of its queries per
// iteration; a run that still searches more than kGiveUpShare of them is handed over to the host-driven loop
// (the exclusion cache costs more than it saves there).
constexpr int kFirstBatch = 4;
constexpr int kBridgeBatch = 2;  // enqueued behind the first batch: covers the host's look at the first batch's state
constexpr double kGiveUpShare = 0.15;

// launch with programmatic stream serialization (see pdl_wait above)
template <class Kernel>
static cudaError_t launch_pdl(Kernel k, int blocks, int threads, size_t smem, cudaStream_t stream, const LoopArgs& a) {
  cudaLaunchConfig_t cfg;
  std::memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)blocks);
  cfg.blockDim = dim3((unsigned)threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, k, a);
}

// Enqueues the kernels of ICP iteration `it` of this call: the search kernel in the cold first iteration (nothing
// cached yet), else the cached pass with its search of the flagged queries; then the finish kernel.
template <int MODE>
static int enqueue_iteration(cb_context* ctx, const LoopArgs& a, int it, int blocks_cold, int blocks_cached) {
  if (it == 0)
    CB_CUDA(launch_pdl(icp_search_kernel<MODE>, blocks_cold, kBlock, 0, ctx->stream, a));
  else
    CB_CUDA(launch_pdl(icp_cached_pipe_kernel<MODE>, blocks_cached, kBlock, sizeof(PipeSmem<MODE == kModeCombined>),
                       ctx->stream, a));
  CB_CUDA(launch_pdl(icp_finish_kernel<MODE>, 1, 32, 0, ctx->stream, a));
  ctx->launches += 2;
  return CB_OK;
}

int icp_loop_estimate(cb_icp* icp, const cb_icp_params* prm, cb_icp_result* res, int* hand_over) {
  *hand_over = 0;
  cb_context* ctx = icp->ctx;
  const uint64_t launches0 = ctx->launches;
  const int max_iter = std::max(prm->max_iter, 0);
  const int timing = prm->timing;
  if (!icp->d_state) CB_TRY(icp->mem.alloc(&icp->d_state, 1));
  if (!icp->h_state) CB_TRY(icp->mem.alloc_host(&icp->h_state, 1));
  while (timing != 0 && (int)icp->events.size() < 2 * max_iter) {
    cudaEvent_t e;
    CB_CUDA(cudaEventCreate(&e));
    icp->events.push_back(e);
  }
  const size_t ns = icp->src->n;
  LoopArgs a;
  std::memset(&a, 0, sizeof(a));
  a.dst = grid_view(icp->dst);
  a.src_pts = icp->src->d_pts;
  a.src_nrm = (prm->metric == CB_ICP_COMBINED) ? icp->src->d_nrm : nullptr;
  a.n_src = (uint32_t)ns;
  a.max_d2 = prm->max_d2;
  a.w_pt = prm->w_pt;
  a.w_pl = prm->w_pl;
  a.wk_pt = prm->pt_weight_kind == CB_WEIGHT_RBF;
  a.wk_pl = prm->pl_weight_kind == CB_WEIGHT_RBF;
  a.wc_pt = prm->pt_weight_coeff;
  a.wc_pl = prm->pl_weight_coeff;
  a.tol = prm->tol;
  for (int r = 0; r < 3; r++) {
    a.dm[r] = icp->dst_mean[r];
    a.src_mean[r] = icp->src_mean[r];
  }
  const bool dst_has_normals = icp->dst->d_nrm != nullptr;
  a.has_pt = prm->w_pt > 0.f;
  a.has_pl = (prm->w_pl > 0.f) && dst_has_normals;
  a.bail = (prm->w_pl > 0.f) && !dst_has_normals;
  a.cache_pos = icp->d_nn_pos;
  a.cache_r = icp->d_nn_d2;
  const float h = 1.0f / a.dst.inv_h;  // cell edge of the destination grid
  a.slack_first = kSlackFirst * h;
  a.slack_min = kSlackMin * h;
  a.slack_max = kSlackMax * h;
  a.st = icp->d_state;
  static const bool trace = getenv("CB_LOOP_TRACE") != nullptr;
  a.trace = trace ? 1 : 0;
  // cold iteration (first launch: nothing cached): search kernel, one 256-query chunk per block; warm iterations:
  // the persistent cached pass (PipeSmem::kT queries per tile), which also searches the queries it flags
  const int blocks_cold = std::max(1, (int)((ns + kBlock - 1) / kBlock));
  // once per device (function attributes belong to the device the context is on, not to the process): the pipeline's
  // dynamic shared memory, the whole shared-memory carveout (4 / 2 blocks of 56 / 98 KB per SM), and how many blocks
  // of the cached pass are resident per SM
  static bool attr_set_dev[64] = {};
  static int resident_dev[64][2] = {};
  bool& attr_set = attr_set_dev[ctx->device & 63];
  int* resident = resident_dev[ctx->device & 63];
  if (!attr_set) {
    CB_CUDA(cudaFuncSetAttribute(icp_cached_pipe_kernel<kModeP2PCentered>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)sizeof(PipeSmem<false>)));
    CB_CUDA(cudaFuncSetAttribute(icp_cached_pipe_kernel<kModeCombined>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)sizeof(PipeSmem<true>)));
    CB_CUDA(cudaFuncSetAttribute(icp_cached_pipe_kernel<kModeP2PCentered>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                 (int)cudaSharedmemCarveoutMaxShared));
    CB_CUDA(cudaFuncSetAttribute(icp_cached_pipe_kernel<kModeCombined>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                 (int)cudaSharedmemCarveoutMaxShared));
    CB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident[0], icp_cached_pipe_kernel<kModeP2PCentered>, kBlock,
                                                          sizeof(PipeSmem<false>)));
    CB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident[1], icp_cached_pipe_kernel<kModeCombined>, kBlock,
                                                          sizeof(PipeSmem<true>)));
    attr_set = true;
  }
  // persistent cached pass: a whole number of resident blocks per SM (never more blocks than tiles)
  const bool p2p = prm->metric == CB_ICP_POINT_TO_POINT;
  const int per_sm = std::max(1, resident[p2p ? 0 : 1]);
  const size_t tile = (size_t)pipe_qpt(!p2p) * kBlock;
  const int blocks_cached = std::max(1, std::min(ctx->sm_count * per_sm, (int)((ns + tile - 1) / tile)));
  CB_TRY(get_reduce_scratch(ctx, blocks_cold, kMaxValues, &a.rs));
  Exchange ex;
  std::memset(&ex, 0, sizeof(ex));
  const bool fused = ctx->world > 1 && arm_exchange(ctx, &ex);  // tables + timeout; the pass number lives in LoopState
  if (fused) ctx->seq -= 1;  // arm_exchange numbered a pass that is not issued here
  if (ctx->world > 1 && !fused) {
    set_error("the device-resident ICP loop needs the fused exchange (cb_comm_ipc_attach) when world > 1");
    return CB_ERR_UNSUPPORTED;
  }
  a.rs.ex = ex;
  ctx->pass_armed = false;

  LoopState* hs = icp->h_state;
  std::memset(hs, 0, sizeof(*hs));
  std::memcpy(hs->T, prm->T_init, sizeof(hs->T));       // icp_base.hpp:71
  std::memcpy(hs->T_prev, prm->T_init, sizeof(hs->T));
  hs->last_delta = INFINITY;
  hs->xseq = ctx->seq;
  CB_CUDA(cudaMemcpyAsync(icp->d_state, hs, sizeof(*hs), cudaMemcpyHostToDevice, ctx->stream));

  int issued = 0;
  // Batches are enqueued ONE AHEAD of the batch whose state the host is looking at: the device never waits for the host
  // between batches (with several ranks such a gap shows up as a peer wait in the next iteration), and the
  // hand-over / convergence decisions lag by at most one batch. Two pinned copies of LoopState alternate.
  if (!icp->h_state2) CB_TRY(icp->mem.alloc_host(&icp->h_state2, 1));
  for (int e = 0; e < 2; ++e)
    if (!icp->batch_ev[e]) CB_CUDA(cudaEventCreateWithFlags(&icp->batch_ev[e], cudaEventDisableTiming));
  LoopState* hbuf[2] = {icp->h_state, icp->h_state2};
  int enq = 0, checked = 0;  // batches enqueued / examined
  auto enqueue_batch = [&](int n) -> int {
    for (int k = 0; k < n; ++k) {
      if (prm->flush_l2) CB_TRY(cb_context_flush_l2(ctx));
      if (timing) CB_CUDA(cudaEventRecord(icp->events[2 * (issued + k)], ctx->stream));
      if (p2p)
        CB_TRY(enqueue_iteration<kModeP2PCentered>(ctx, a, issued + k, blocks_cold, blocks_cached));
      else
        CB_TRY(enqueue_iteration<kModeCombined>(ctx, a, issued + k, blocks_cold, blocks_cached));
      if (timing) CB_CUDA(cudaEventRecord(icp->events[2 * (issued + k) + 1], ctx->stream));
    }
    CB_CUDA(cudaGetLastError());
    issued += n;
    CB_CUDA(cudaMemcpyAsync(hbuf[enq & 1], icp->d_state, sizeof(LoopState), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaEventRecord(icp->batch_ev[enq & 1], ctx->stream));
    ++enq;
    return CB_OK;
  };
  bool stop = false, give_up = false;
  if (max_iter > 0) CB_TRY(enqueue_batch(std::min(kFirstBatch, max_iter)));
  while (checked < enq) {
    // (a short bridge batch until the first state has been examined: a run that is given up then costs two more device
    // iterations, not a full batch)
    if (!stop && issued < max_iter && enq - checked < 2)
      CB_TRY(enqueue_batch(std::min(checked == 0 ? kBridgeBatch : kBatch, max_iter - issued)));
    CB_CUDA(cudaEventSynchronize(icp->batch_ev[checked & 1]));
    hs = hbuf[checked & 1];
    ++checked;
    if (hs->done != 0 || issued >= max_iter) {
      stop = true;  // converged / failed (launches already enqueued return at once) or everything is enqueued
    } else if (hs->iters >= kFirstBatch && hs->searched_all > kGiveUpShare * hs->queries_all) {
      stop = true;  // not converging: no further batch; the one already in flight (if any) still completes
      give_up = true;
    }
  }
  if (give_up && hs->done == 0 && hs->iters < max_iter) *hand_over = 1;
  if (max_iter == 0) CB_CUDA(cudaStreamSynchronize(ctx->stream));
  ctx->seq = hs->xseq;
  if (hs->done == 2) {
    set_error("device-resident ICP loop: a peer rank did not deliver its row in time (rank %d of %d, iteration %d)",
              ctx->rank, ctx->world, hs->iters);
    ctx->ex_ready = false;
    return hs->error ? hs->error : CB_ERR_NCCL;
  }
  const int iters = hs->iters;
  if (trace) {
    unsigned long long prev = 0;
    for (int k = std::max(0, iters - 64); k < iters; ++k) {
      const unsigned long long* t = hs->trace[k & 63];
      fprintf(stderr, "[rank %d iteration %d] searched %llu of %zu queries; start->last warp at the reduction %.1f us, ->reduced %.1f us, ->peers %.1f us, ->solved %.1f us; period %.1f us\n",
              ctx->rank, k, t[4], ns, (t[5] - t[0]) * 1e-3, (t[1] - t[5]) * 1e-3, (t[2] - t[1]) * 1e-3, (t[3] - t[2]) * 1e-3,
              prev ? (t[0] - prev) * 1e-3 : 0.0);
      prev = t[0];
    }
  }
  icp->iter_ms.assign(iters, 0.0);
  double total = 0;
  for (int k = 0; k < iters && timing != 0; k++) {
    float ms = 0.f;
    CB_CUDA(cudaEventElapsedTime(&ms, icp->events[2 * k], icp->events[2 * k + 1]));
    icp->iter_ms[k] = ms;
    total += ms;
  }
  icp->search_ms = total;
  icp->nn_valid = iters > 0;
  icp->nn_stored = false;  // d_nn_pos / d_nn_d2 hold the cache, not a per-query result list
  icp->warm_ok = false;
  icp->engine_last = false;
  icp->loop_last = true;
  icp->searched_last = hs->searched_last;
  std::memcpy(icp->T_search, hs->T_prev, sizeof(icp->T_search));
  icp->max_d2_search = prm->max_d2;
  std::memcpy(res->T, hs->T, sizeof(res->T));
  res->iterations = iters;
  res->last_delta = hs->last_delta;
  res->converged = hs->last_delta < prm->tol;
  res->num_corr = (uint64_t)(hs->n_corr + 0.5);
  res->gpu_ms_total = total;
  res->gpu_ms_search = total;
  res->kernel_launches = ctx->launches - launches0;
  return CB_OK;
}

}  // namespace cb
