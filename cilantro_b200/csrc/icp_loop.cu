// Device-resident rigid ICP loop (product code, sm_90a).
//
// IterativeClosestPointBase::estimate() (registration/icp_base.hpp:68-87) for the default correspondence engine:
// TWO kernels per ICP iteration and NO host round trip between iterations. In iteration k the first kernel
//   1. reads the current estimate T_k from device memory (LoopState),
//   2. finds every source point's correspondence under T_k (below),
//   3. accumulates the estimator's moments, reduces them warp -> block and writes one row per block;
// the finish kernel (one block, launched behind it)
//   4. folds the block rows into this GPU's 16 / 28 totals in a fixed order, all-reduces them with the peer ranks
//      over NVLink peer memory (reduce.cuh, bounded wait), then solves on the device — Kabsch / one Gauss-Newton
//      step, rotation() re-orthonormalisation, compose, update norm, convergence test (solve_core.hpp; the same code
//      the host loop runs) — and writes T_{k+1} back to LoopState.
// The host enqueues the launches back to back and reads LoopState once per batch; launches after convergence
// return at once. With several ranks every rank solves the same totals redundantly -> bit-identical transforms.
//
// Correspondences WITHOUT a search (exact). Every search also returns an EXCLUSION bound: a radius r such that
// every reference point other than the match is at least r away from the query (warp_search_wide.cuh). The next
// iteration moves the query by delta = |T_{k+1} s - T_k s|, so every other point is still at least r - delta away
// (triangle inequality); if the cached match's distance under T_{k+1} — evaluated with the contract arithmetic,
// i.e. the very number the search would compute for it — is below that, the match is provably still the unique
// nearest neighbour and its (index, d2) is what the full search would return, bit for bit. Only the queries
// that fail the test are searched again, inside the same pass: each warp lists the ones it flagged and searches them
// after its last tile, on dense warps. All bounds are rounded conservatively (directed rounding + 2^-18 relative
// margins, far above the 6-ulp error of the fp32 distance evaluation); an exact tie can never pass the strict test.
// As ICP converges the per-iteration motion shrinks geometrically and almost every query takes the cached path:
// the iteration becomes one streaming pass (12 B query + 8 B cache + one 12 B gather per source point).
//
// With a projection attached (cb_icp_set_projection, DESIGN §4.21) the first kernel is icp_projective_kernel instead:
// every source point looks up the one destination point its pixel shows, with no cache and no search.
#include "cache_rule.hpp"
#include "icp_accumulate.cuh"
#include "icp_kernels.cuh"
#include "icp_object.hpp"
#include "launch.cuh"
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
  // cached pass: packed xyz (12 B per point, same order) of src_pts (padded to whole 32-query windows), of dst.pts and
  // of dst.nrm (nullptr unless the plane term is on): the bytes it streams and gathers, without the unread .w
  const float* src_xyz;
  const float* dst_xyz;
  const float* dst_nxyz;
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
  uint32_t* flagged;       // cached pass: per warp of its grid, the queries it flagged, ascending (flagged_per_warp each)
  uint32_t flagged_per_warp;
  LoopState* st;
  ReduceScratch rs;
  uint32_t rows;  // block rows of the pass in rs.partials (its grid size)
  int trace;      // CB_LOOP_TRACE: fill LoopState::trace
  // projective search (icp_projective_kernel): the index map (sorted dst positions, -1 empty) and its projection
  const int* proj_map;
  Projection prj;
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
// (icp_finish_kernel): inside the search kernel its temporaries were spilled at that kernel's register budget, and a
// local-memory word of ONE thread lives in its own 128-byte line - after a 10 M-point pass every one of them was a
// cold DRAM miss (in a %globaltimer trace the solve took many times its arithmetic). So nothing here may be indexed
// at run time (solve_core.hpp picks by selects): the solve keeps its temporaries in registers.
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

// Lanes per queued region in the wide search's pooled scan (warp_search_wide.cuh). The cold pass keeps one lane per
// region. The cached pass's search uses pairs of lanes: its region scan then needs fewer live registers (DESIGN §4.2).
constexpr unsigned int kColdGroup = 1, kWarmGroup = 2;
// The query failed the exclusion test: its cached match seeds the search and its last motion sets the slack.
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
    float ox, oy, oz;
    rule::transform_point(cx.Tp, s.x, s.y, s.z, ox, oy, oz);
    const float ex = __fsub_rn(cp.qx, ox), ey = __fsub_rn(cp.qy, oy), ez = __fsub_rn(cp.qz, oz);
    const float dl = __fsqrt_ru(__fmaf_ru(ez, ez, __fmaf_ru(ey, ey, __fmul_ru(ex, ex))));
    // the next step is expected to be about half of this one, and a hit needs r - (motion) > d: widen by 2 x
    slack = fminf(fmaxf(__fmul_rn(2.f, dl), a.slack_min), a.slack_max);
    sd = a.cache_pos[cp.i];
  }
  const WideBest wb = warp_grid_nearest_wide<kWarmGroup>(a.dst, *wsm, act, cp.qx, cp.qy, cp.qz, a.max_d2, sd, slack);
  if (act) {
    cp.pos = (wb.idx >= 0 && wb.d2 < a.max_d2) ? wb.pos : -1;
    cp.d2 = wb.d2;
    a.cache_pos[cp.i] = cp.pos;
    a.cache_r[cp.i] = rule::cache_radius(wb.D2);
  }
  return cp;
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
// Elementwise over the source cloud: per query 12 B (point) + 8 B (cache) streamed and one 12 B gather of the cached
// match (+ 12 B normal for the plane term), all from packed xyz copies (LoopArgs::src_xyz, dst_xyz, dst_nxyz): the
// float4 arrays' .w holds index bits this pass never reads. Queries that pass the exclusion test accumulate their pair
// at once. The others are searched by the warp that flagged them, after its last tile: after each 32-query slot the
// warp's ballot appends the flagged query indices, in ascending order, to the warp's list in global memory
// (a.flagged); once the warp's copies have drained it searches the list lane-dense, 32 at a time (search_chunk_body: same slack rule, warm
// seed and cache update as the cold search), in its own pipeline buffers, and the searching lane adds its pair to the
// warp's sums. Only __syncwarp is involved, so a searching warp holds up no other warp of its block. A converged
// iteration flags a few dozen of 10^6 queries: the search gets no shared memory of its own and no call site inside the
// streaming loop, whose registers it would otherwise share.
// PERSISTENT: the grid is a whole number of resident blocks per SM, a block walks the tiles blockIdx.x, + gridDim.x,
// ... (static round-robin: every tile costs the same, and the assignment — hence, with the fixed list order, the
// summation order — is fixed), the next tiles' loads are in flight while the current tile is evaluated, and the
// moments are reduced ONCE per block (a per-tile reduction cost as much as the tile itself). Every block writes its row
// to rs.partials (zeros included: the finish kernel folds every row) and is done.
// The loads are not staged in registers: a register-staged version needed 128 registers -> 2 blocks/SM, few warp
// slots occupied, long-scoreboard stalls on top - each thread can only keep the loads in flight that it has registers
// for. Here every thread runs a private pipeline of cp.async copies into shared memory (LDGSTS: no destination
// register, no scoreboard slot), kDepthA tiles of stage A and kDepthB of stage B:
//   stage A (tile k+kDepthA-1)  the streamed arrays: the warp's 32 query points as one contiguous 384-byte window of
//                               packed xyz (24 lanes x 16 B), then per lane the exclusion radius (4 B) and cached match
//                               (4 B)
//   stage B (tile k+kDepthB-1)  the gathers, once A has landed: the matched destination point (+ normal for the plane
//                               term), 3 x 4 B each
//   stage C (tile k)            evaluation from shared memory; a lane reads its point at stride 3 floats (no bank
//                               conflict)
// Stage B reads only what its own lane copied in stage A. The query points are the one thing a lane reads from other
// lanes' copies: so a __syncwarp follows each cp.async.wait_group before stage C, and another one after stage C keeps
// the next step's stage A from overwriting a window a lane is still reading. There is no block barrier inside the tile
// loop. The buffers are laid out warp by warp (WarpPipe), so a warp whose copies have drained owns one contiguous
// region, and its search buffer (WideSearchSmem) lives there.
//   p2p: 256-query tiles (one query per thread), stage A 4 deep and stage B 3 deep: each gather is issued two tiles
//        ahead of its evaluation. 29 KB of pipeline, 4 blocks per SM (64 registers).
//   combined: 512-query tiles, stage A 3 deep and stage B 2 deep: 54 KB of pipeline, 2 blocks per SM (128 registers).
//        At 3 blocks (80 registers, 256-query tiles) the exclusion test and the 28 accumulators spilled on every query.
// (DESIGN §4.2 has the measured alternatives.)
__host__ __device__ constexpr int pipe_qpt(bool normals) { return normals ? 2 : 1; }
__host__ __device__ constexpr int pipe_depth_a(bool normals) { return normals ? 3 : 4; }
__host__ __device__ constexpr int pipe_depth_b(bool normals) { return normals ? 2 : 3; }
__host__ __device__ constexpr int pipe_min_blocks(bool normals) { return normals ? 2 : 4; }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async_16_cg(void* dst_smem, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_4(void* dst_smem, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// a query's cached exclusion radius and match, side by side: one 8-byte shared load
struct alignas(8) RadiusSeed {
  float r;
  int seed;
};
// One warp's pipeline buffers: entry e = k * 32 + lane belongs to the warp's k-th query of a tile on that lane; the
// packed xyz arrays hold its coordinates at 3 e, 3 e + 1, 3 e + 2 (src[.][k * 96 ...] is one 16-byte aligned window).
template <bool kNormals>
struct alignas(16) WarpPipe {
  static constexpr int kA = pipe_depth_a(kNormals), kB = pipe_depth_b(kNormals);
  static constexpr int kW = pipe_qpt(kNormals) * 32;  // the warp's queries per tile
  float src[kA][3 * kW];
  RadiusSeed rs[kA][kW];
  float pt[kB][3 * kW];
  float nr[kNormals ? kB : 1][kNormals ? 3 * kW : 1];
};
template <bool kNormals>
struct PipeSmem {
  WarpPipe<kNormals> warp[kBlock / 32];
};
static_assert(sizeof(WideSearchSmem) <= sizeof(WarpPipe<false>) && sizeof(WideSearchSmem) <= sizeof(WarpPipe<true>),
              "a warp's search buffer lives in its drained pipeline region");

template <int MODE>
__global__ void __launch_bounds__(kBlock, pipe_min_blocks(MODE == kModeCombined)) icp_cached_pipe_kernel(const __grid_constant__ LoopArgs a) {
  constexpr int NV = (MODE == kModeP2PCentered) ? kP2PValues : kCombinedValues;
  constexpr bool kNormals = (MODE == kModeCombined);
  constexpr int kQpt = pipe_qpt(kNormals), kTile = kQpt * kBlock;
  // stage A of tile n + kLeadA and stage B of tile n + kLeadB are issued while tile n is evaluated
  constexpr int kDepthA = pipe_depth_a(kNormals), kDepthB = pipe_depth_b(kNormals);
  constexpr int kLeadA = kDepthA - 1, kLeadB = kDepthB - 1;
  static_assert(kLeadB >= 1 && kLeadA > kLeadB, "a gather needs its stream landed one step earlier");
  extern __shared__ __align__(16) unsigned char pipe_raw[];
  __shared__ BlockCtx cx;
  __shared__ AsyncReduceSmem<NV> rsm;
  const unsigned int tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  WarpPipe<kNormals>& wp = reinterpret_cast<PipeSmem<kNormals>*>(pipe_raw)->warp[warp];
  const uint32_t ntiles = (a.n_src + kTile - 1) / kTile;
  const bool want_nrm = kNormals && a.has_pl != 0;

  // stage A of tile `tile` into buffer `buf`: nothing here depends on the loop state
  auto stage_a = [&](uint32_t tile, int buf) {
    if (tile < ntiles) {
#pragma unroll
      for (int k = 0; k < kQpt; k++) {
        // the warp's window: queries w0 .. w0 + 31 (src_xyz is padded to whole windows)
        const uint32_t w0 = tile * kTile + k * kBlock + warp * 32u, i = w0 + lane;
        if (w0 < a.n_src && lane < 24u)
          cp_async_16_cg(&wp.src[buf][k * 96 + 4 * lane], a.src_xyz + (size_t)w0 * 3u + 4u * lane);
        if (i < a.n_src) {
          cp_async_4(&wp.rs[buf][k * 32 + lane].r, a.cache_r + i);
          cp_async_4(&wp.rs[buf][k * 32 + lane].seed, a.cache_pos + i);
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
        const uint32_t e = k * 32 + lane, i = tile * kTile + k * kBlock + tid;
        if (i < a.n_src) {
          const RadiusSeed cs = wp.rs[abuf][e];
          if (cs.seed >= 0 && cs.r > 0.f) {
            const int sd = cs.seed;
            const float* p = a.dst_xyz + (size_t)sd * 3u;
#pragma unroll
            for (int c = 0; c < 3; c++) cp_async_4(&wp.pt[bbuf][3 * e + c], p + c);
            if (kNormals && want_nrm) {
              const float* nv = a.dst_nxyz + (size_t)sd * 3u;
#pragma unroll
              for (int c = 0; c < 3; c++) cp_async_4(&wp.nr[kNormals ? bbuf : 0][3 * e + c], nv + c);
            }
          }
        }
      }
    }
    cp_async_commit();
  };

  const uint32_t t0 = blockIdx.x, stride = gridDim.x;
  // Step n of the block (n = -kLeadA, -kLeadA + 1, ...) commits two groups, A(n + kLeadA) then B(n + kLeadB) (either
  // may be empty), and evaluates tile n once it is >= 0. With that fixed order, A(n + kLeadB) has landed when at most
  // 2 (kLeadA - kLeadB) groups are pending after A(n + kLeadA), and B(n) when at most 2 kLeadB are pending after
  // B(n + kLeadB).
  // The dependency wait comes BEFORE the first copies: the cache arrays are rewritten every iteration, their 4-byte
  // copies go through L1 (cp.async.ca), and only accesses after griddepcontrol.wait are guaranteed to see the previous
  // kernels' writes. What programmatic launch buys here: the blocks are resident when the finish kernel ends, and the
  // one-block finish kernel of this iteration, released at once, is resident and waiting when this grid drains.
  pdl_wait();
  pdl_launch_dependents();
#pragma unroll
  for (int n = 0; n < kLeadA - kLeadB; n++) {  // steps -kLeadA .. -kLeadB - 1: no gather due yet
    stage_a(t0 + n * stride, n);
    cp_async_commit();
  }
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
#pragma unroll
  for (int n = kLeadA - kLeadB; n < kLeadA; n++) {  // steps -kLeadB .. -1
    stage_a(t0 + n * stride, n);
    cp_async_wait<2 * (kLeadA - kLeadB)>();
    stage_b(t0 + (n - (kLeadA - kLeadB)) * stride, n - (kLeadA - kLeadB), n - (kLeadA - kLeadB));
  }
  double acc[NV];
#pragma unroll
  for (int v = 0; v < NV; v++) acc[v] = 0.0;
  // the warp's row of the block reduction: what the warp folded before its searches, then their pairs. (The fold adds
  // value by value: the transposing butterfly of warp_sum_to_slot<16, false> keeps acc[] in local memory.)
  if (lane < NV) rsm.slot[warp][lane] = 0.0;
  // the warp's flagged queries, ascending; `flagged` is warp-uniform
  uint32_t* const list = a.flagged + (size_t)(blockIdx.x * (kBlock / 32) + warp) * a.flagged_per_warp;
  unsigned int flagged = 0;
  // step n evaluates tile t0 + n*stride from A buffer n % kDepthA and B buffer n % kDepthB
  int abuf = 0, bbuf = 0;
#pragma unroll 1
  for (uint32_t tile = t0; tile < ntiles; tile += stride) {
    const int abuf_next = (abuf == kDepthA - 1) ? 0 : abuf + 1, bbuf_next = (bbuf == kDepthB - 1) ? 0 : bbuf + 1;
    // A(n + kLeadA) goes where tile n - 1 was, A(n + kLeadB) is in buffer (n + kLeadB) % kDepthA, and B(n + kLeadB)
    // goes where tile n - 1's gathers were
    const int abuf_prev = (abuf == 0) ? kDepthA - 1 : abuf - 1, bbuf_prev = (bbuf == 0) ? kDepthB - 1 : bbuf - 1;
    const int abuf_b = (abuf + kLeadB) % kDepthA;
    stage_a(tile + kLeadA * stride, abuf_prev);
    cp_async_wait<2 * (kLeadA - kLeadB)>();
    stage_b(tile + kLeadB * stride, abuf_b, bbuf_prev);
    cp_async_wait<2 * kLeadB>();
    __syncwarp();  // the other lanes' copies of this tile's query windows have landed too
    const uint32_t base = tile * kTile;
#pragma unroll
    for (int k = 0; k < kQpt; k++) {
      const uint32_t e = k * 32 + lane, i = base + k * kBlock + tid;
      const bool active = i < a.n_src;
      bool miss = active;
      if (active) {
        const RadiusSeed cs = wp.rs[abuf][e];
        const float rc = cs.r;
        const int sd = cs.seed;
        if (rc > 0.f) {
          const float* sc = &wp.src[abuf][3 * e];
          // the exclusion test (cache_rule.hpp): hit -> the cached match is this iteration's exact search result
          rule::Verdict v;
          float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
          rule::cached_match_test(
              cx.T, cx.Tp, sc[0], sc[1], sc[2], rc, sd, a.max_d2,
              [&] { return make_float4(wp.pt[bbuf][3 * e], wp.pt[bbuf][3 * e + 1], wp.pt[bbuf][3 * e + 2], 0.f); }, p, v);
          miss = v.miss;
          if (!miss) a.cache_r[i] = v.r2;
          if (v.pair) {
            const float* nv = &wp.nr[kNormals ? bbuf : 0][kNormals ? 3 * e : 0];
            accumulate_pair<MODE, true>(
                acc, cx, a.has_pt != 0, a.has_pl != 0, p, v.qx, v.qy, v.qz, a.src_nrm != nullptr,
                [&] { return kNormals ? make_float4(nv[0], nv[1], nv[2], 0.f) : make_float4(0.f, 0.f, 0.f, 0.f); },
                [&] { return __ldg(a.src_nrm + i); }, v.d2);
          }
        }
      }
      // flagged queries -> the warp's list, in ascending order
      const unsigned int mm = __ballot_sync(0xffffffffu, miss);
      if (miss) list[flagged + __popc(mm & ((1u << lane) - 1u))] = i;
      flagged += __popc(mm);
    }
    __syncwarp();  // every lane has read this tile's windows before the next step's stage A reuses the buffer
    abuf = abuf_next;
    bbuf = bbuf_next;
  }
  cp_async_wait<0>();
  // the warp's copies have drained (its pipeline region is free for the search) and its list entries are visible to
  // all of its lanes
  __syncwarp();
  // The warp searches its list, 32 queries at a time; the searching lane accumulates its pair. Before each search the
  // accumulators are folded into the warp's row and restart from zero, so that none of them is live across it.
  WideSearchSmem* wsm = reinterpret_cast<WideSearchSmem*>(&wp);
  for (unsigned int c = 0; c < flagged; c += 32u) {
    warp_sum_to_slot<NV, true>(acc, rsm);
#pragma unroll
    for (int v = 0; v < NV; v++) acc[v] = 0.0;
    const bool act = c + lane < flagged;
    const ChunkPair cp = search_chunk_body(a, cx, wsm, act, act ? list[c + lane] : 0u);
    if (cp.pos >= 0) {
      const float4 dp = __ldg(a.dst.pts + cp.pos);
      accumulate_pair<MODE, true>(
          acc, cx, a.has_pt != 0, a.has_pl != 0, dp, cp.qx, cp.qy, cp.qz, a.src_nrm != nullptr,
          [&] { return __ldg(a.dst.nrm + cp.pos); }, [&] { return __ldg(a.src_nrm + cp.i); }, cp.d2);
    }
  }
  if (lane == 0 && flagged > 0u) {
    atomicAdd(&a.st->searched_cur, (unsigned long long)flagged);
    if (a.trace) atomicAdd(&a.st->trace[__ldcg(&a.st->iters) & 63][4], (unsigned long long)flagged);
  }
  warp_sum_to_slot<NV, true>(acc, rsm);
  if (a.trace && lane == 0) atomicMax(&a.st->trace[__ldcg(&a.st->iters) & 63][5], global_timer_ns());
  double row;
  if (block_row_from_slots<NV>(rsm, row) && lane < NV) a.rs.partials[(size_t)blockIdx.x * NV + lane] = row;
}

// ---- kernel 1 of the cold iteration (the first of a call: nothing cached yet): every query searched -------------
// PERSISTENT, like the cached pass: the grid is a whole number of resident blocks per SM, and each warp walks the
// 32-query chunks of the cell-sorted source round-robin (warp w of the grid takes chunks w, w + W, ..., W = the grid's
// warps), so the assignment and the summation order are fixed. Each chunk is one lane-dense wide search (kColdGroup
// lanes per region); the searching lane updates the cache and accumulates its pair, and the warp folds its pairs into
// its row of the block reduction after every chunk, so none of the accumulators is live across a search. The next
// chunk's source points are loaded before the current chunk's search. The last warp of the block writes the block row
// to rs.partials, which the finish kernel folds: a few hundred rows instead of one per 256 queries.
// Register budget: p2p 64 registers, 4 blocks per SM. The combined metric's 28 accumulators spilled at 64 registers
// (its 10 M cold iteration took 1.97 ms against 1.69 ms at 80 registers, 3 blocks per SM; DESIGN §4.2).
__host__ __device__ constexpr int cold_min_blocks(bool combined) { return combined ? 3 : 4; }

template <int MODE>
__global__ void __launch_bounds__(kBlock, cold_min_blocks(MODE == kModeCombined))
    icp_search_kernel(const __grid_constant__ LoopArgs a) {
  constexpr int NV = (MODE == kModeP2PCentered) ? kP2PValues : kCombinedValues;
  __shared__ BlockCtx cx;
  __shared__ WideSearchSmem wsm[kBlock / 32];
  __shared__ AsyncReduceSmem<NV> rsm;
  const unsigned int tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const uint32_t nchunks = (a.n_src + 31u) / 32u;
  const uint32_t c0 = blockIdx.x * (kBlock / 32) + warp, stride = gridDim.x * (kBlock / 32);
  auto load_src = [&](uint32_t chunk) {
    const uint32_t i = chunk * 32u + lane;
    return (chunk < nchunks && i < a.n_src) ? __ldg(a.src_pts + i) : make_float4(0.f, 0.f, 0.f, 0.f);
  };

  pdl_wait();               // the state of the previous finish kernel
  pdl_launch_dependents();  // the finish kernel may be scheduled now and wait for this grid to drain
  float4 s_next = load_src(c0);
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
  if (lane < NV) rsm.slot[warp][lane] = 0.0;
  unsigned int searched = 0;
#pragma unroll 1
  for (uint32_t chunk = c0; chunk < nchunks; chunk += stride) {
    const uint32_t i = chunk * 32u + lane;
    const bool act = i < a.n_src;
    const float4 s = s_next;
    s_next = load_src(chunk + stride);
    float qx = 0.f, qy = 0.f, qz = 0.f;
    if (act) rule::transform_point(cx.T, s.x, s.y, s.z, qx, qy, qz);
    const WideBest wb = warp_grid_nearest_wide<kColdGroup>(a.dst, wsm[warp], act, qx, qy, qz, a.max_d2, -1, a.slack_first);
    double acc[NV];
#pragma unroll
    for (int v = 0; v < NV; v++) acc[v] = 0.0;
    if (act) {
      const int pos = (wb.idx >= 0 && wb.d2 < a.max_d2) ? wb.pos : -1;
      a.cache_pos[i] = pos;
      a.cache_r[i] = rule::cache_radius(wb.D2);
      if (pos >= 0) {
        const float4 dp = __ldg(a.dst.pts + pos);
        accumulate_pair<MODE, true>(
            acc, cx, a.has_pt != 0, a.has_pl != 0, dp, qx, qy, qz, a.src_nrm != nullptr,
            [&] { return __ldg(a.dst.nrm + pos); }, [&] { return __ldg(a.src_nrm + i); }, wb.d2);
      }
    }
    warp_sum_to_slot<NV, true>(acc, rsm);
    searched += (uint32_t)__popc(__ballot_sync(0xffffffffu, act));
  }
  if (lane == 0 && searched > 0u) {
    atomicAdd(&a.st->searched_cur, (unsigned long long)searched);
    if (a.trace) atomicAdd(&a.st->trace[trace_slot][4], (unsigned long long)searched);
  }
  if (a.trace && lane == 0) atomicMax(&a.st->trace[trace_slot][5], global_timer_ns());
  double row;
  if (block_row_from_slots<NV>(rsm, row) && lane < NV) a.rs.partials[(size_t)blockIdx.x * NV + lane] = row;
}

// ---- kernel 1 of a projective iteration: project, look up, accumulate ------------------------------------------------
// find_correspondences_ of CorrespondenceSearchProjective (DESIGN §4.21) fused with the accumulation. PERSISTENT and
// grid-stride over the cell-sorted source, so the assignment and the summation order are fixed: per query the packed
// point (12 B), one map read (4 B), and for a pixel that shows a destination point its packed coordinates (12 B) and,
// with the plane term, its normal (12 B); the symmetric metric adds the source normal. Nothing is cached, nothing is
// searched: searched_cur stays 0, so the loop never hands the run over.
// Register budget (__launch_bounds__ caps): p2p at most 64 registers for 4 blocks per SM (it uses 64); combined at most 128
// for 2 blocks per SM (it uses 108; at the 80-register cap of 3 blocks its 28 accumulators spilled).
__host__ __device__ constexpr int proj_min_blocks(bool combined) { return combined ? 2 : 4; }

template <int MODE>
__global__ void __launch_bounds__(kBlock, proj_min_blocks(MODE == kModeCombined))
    icp_projective_kernel(const __grid_constant__ LoopArgs a) {
  constexpr int NV = (MODE == kModeP2PCentered) ? kP2PValues : kCombinedValues;
  __shared__ BlockCtx cx;
  __shared__ AsyncReduceSmem<NV> rsm;
  const unsigned int tid = threadIdx.x, lane = tid & 31u;
  pdl_wait();               // the state of the previous finish kernel
  pdl_launch_dependents();  // the finish kernel may be scheduled now and wait for this grid to drain
  if (tid == 0) {
    rsm.arrived = 0u;
    load_block_ctx(a, cx);
  }
  __syncthreads();
  if (cx.done) return;  // converged (or failed) in an earlier launch of this batch
  // (the fold adds value by value into zeroed slots: the transposing butterfly of warp_sum_to_slot<16, false> would
  // keep acc[] in local memory)
  if (lane < NV) rsm.slot[tid >> 5][lane] = 0.0;
  __syncwarp();  // the zeroed slots are visible to lane 0's read-modify-write in warp_sum_to_slot
  double acc[NV];
#pragma unroll
  for (int v = 0; v < NV; v++) acc[v] = 0.0;
#pragma unroll 1
  for (uint32_t i = blockIdx.x * kBlock + tid; i < a.n_src; i += gridDim.x * kBlock) {
    const float* s = a.src_xyz + (size_t)i * 3u;
    float qx, qy, qz;
    rule::transform_point(cx.T, __ldg(s), __ldg(s + 1), __ldg(s + 2), qx, qy, qz);
    uint32_t px, py;
    float cz;
    if (!project_pixel(a.prj, qx, qy, qz, px, py, cz)) continue;
    const int pos = __ldg(a.proj_map + (size_t)py * a.prj.w + px);
    if (pos < 0) continue;
    const float* p = a.dst_xyz + (size_t)pos * 3u;
    const float4 dp = make_float4(__ldg(p), __ldg(p + 1), __ldg(p + 2), 0.f);
    const float d2 = rule::contract_d2(qx, qy, qz, dp.x, dp.y, dp.z);
    if (!(d2 < a.max_d2)) continue;
    accumulate_pair<MODE, true>(
        acc, cx, a.has_pt != 0, a.has_pl != 0, dp, qx, qy, qz, a.src_nrm != nullptr,
        [&] {
          const float* n = a.dst_nxyz + (size_t)pos * 3u;
          return make_float4(__ldg(n), __ldg(n + 1), __ldg(n + 2), 0.f);
        },
        [&] { return __ldg(a.src_nrm + i); }, d2);
  }
  warp_sum_to_slot<NV, true>(acc, rsm);
  double row;
  if (block_row_from_slots<NV>(rsm, row) && lane < NV) a.rs.partials[(size_t)blockIdx.x * NV + lane] = row;
}

// ---- kernel 2 of an iteration: fold + exchange + solve (one block) -----------------------------------------------------
// The pass's block rows (a.rows of them) -> this GPU's totals (block_fold_rows: the whole block, in the fixed order of
// the grid reduction) -> all-reduce with the
// peer ranks over NVLink peer memory (reduce.cuh, bounded wait; every rank sums the rows in rank order ->
// bit-identical totals) -> Kabsch / Gauss-Newton step, rotation(), compose, convergence test -> LoopState for the next
// iteration's kernels. Everything after the fold runs in warp 0.
template <int MODE>
__global__ void __launch_bounds__(kBlock, 1) icp_finish_kernel(const __grid_constant__ LoopArgs a) {
  constexpr int NV = (MODE == kModeP2PCentered) ? kP2PValues : kCombinedValues;
  __shared__ BlockCtx cx;
  __shared__ double sbuf[kCombinedValues + 8];
  static_assert(NV + 2 <= kExchangeVals, "row of the fused exchange");
  const unsigned int lane = threadIdx.x;
  // griddepcontrol.wait returns once the whole grid before (cached pass or cold pass) has completed and its
  // rows are visible; it also orders this kernel after the state of the previous iteration
  pdl_wait();
  pdl_launch_dependents();  // the next iteration's cached pass may start streaming
  if (threadIdx.x == 0) load_block_ctx(a, cx);
  __syncthreads();
  if (cx.done) return;
  block_fold_rows<NV>(a.rs.partials, a.rows, sbuf);
  if (threadIdx.x >= 32) return;
  __syncwarp();
  const int trace_slot = a.trace ? (__ldcg(&a.st->iters) & 63) : 0;
  if (a.trace && lane == 0) a.st->trace[trace_slot][1] = global_timer_ns();
  // lanes < NV: the moments; lane NV: queries this rank searched in this iteration; lane NV + 1: its source points
  // (both ride along so that every rank sees the same global search share: the hand-over decision of the host)
  double tot = (lane < NV) ? sbuf[lane] : 0.0;
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

// The cached pass's packed copies: out[3 i .. 3 i + 2] = in[i].xyz for i < n, zeros for n <= i < n_out.
__global__ void pack_xyz_kernel(const float4* __restrict__ in, size_t n, size_t n_out, float* __restrict__ out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_out; i += (size_t)gridDim.x * blockDim.x) {
    const float4 p = i < n ? __ldg(in + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    out[3 * i] = p.x;
    out[3 * i + 1] = p.y;
    out[3 * i + 2] = p.z;
  }
}

int pack_xyz(cb_context* ctx, DeviceScope& mem, const float4* in, size_t n, size_t n_out, float** out) {
  CB_TRY(mem.alloc(out, 3 * std::max<size_t>(n_out, 1)));
  return launch(ctx, pack_xyz_kernel, grid_for(ctx, n_out, kBlock), kBlock, 0, in, n, n_out, *out);
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

// Enqueues the kernels of ICP iteration `it` of this call, with programmatic stream serialization (see pdl_wait
// above): the cold pass in the first iteration (nothing cached yet), else the cached pass with its search of the
// flagged queries; with a projection the projective pass in every iteration; then the finish kernel.
template <int MODE>
static int enqueue_iteration(cb_context* ctx, const LoopArgs& args, int it, int blocks_cold, int blocks_cached,
                             int blocks_proj) {
  LoopArgs a = args;
  // each block of any pass writes one row
  a.rows = (uint32_t)(a.proj_map ? blocks_proj : it == 0 ? blocks_cold : blocks_cached);
  if (a.proj_map)
    CB_TRY(launch_pdl(ctx, icp_projective_kernel<MODE>, blocks_proj, kBlock, 0, a));
  else if (it == 0)
    CB_TRY(launch_pdl(ctx, icp_search_kernel<MODE>, blocks_cold, kBlock, 0, a));
  else
    CB_TRY(launch_pdl(ctx, icp_cached_pipe_kernel<MODE>, blocks_cached, kBlock, sizeof(PipeSmem<MODE == kModeCombined>),
                      a));
  return launch_pdl(ctx, icp_finish_kernel<MODE>, 1, kBlock, 0, a);
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
  // the cached pass's packed copies, once per ICP object (the clouds' index arrays do not change after they are built)
  if (!icp->d_loop_src_xyz) CB_TRY(pack_xyz(ctx, icp->mem, icp->src->d_pts, ns, (ns + 31) / 32 * 32, &icp->d_loop_src_xyz));
  if (!icp->d_loop_dst_xyz) CB_TRY(pack_xyz(ctx, icp->mem, icp->dst->d_pts, icp->dst->n, icp->dst->n, &icp->d_loop_dst_xyz));
  if (a.has_pl && !icp->d_loop_dst_nxyz)
    CB_TRY(pack_xyz(ctx, icp->mem, icp->dst->d_nrm, icp->dst->n, icp->dst->n, &icp->d_loop_dst_nxyz));
  a.src_xyz = icp->d_loop_src_xyz;
  a.dst_xyz = icp->d_loop_dst_xyz;
  a.dst_nxyz = a.has_pl ? icp->d_loop_dst_nxyz : nullptr;
  const float h = 1.0f / a.dst.inv_h;  // cell edge of the destination grid
  a.slack_first = kSlackFirst * h;
  a.slack_min = kSlackMin * h;
  a.slack_max = kSlackMax * h;
  a.st = icp->d_state;
  static const bool trace = getenv("CB_LOOP_TRACE") != nullptr;
  a.trace = trace ? 1 : 0;
  // cold iteration (first launch: nothing cached): the persistent cold pass (32-query chunks per warp); warm
  // iterations: the persistent cached pass (pipe_qpt x kBlock queries per tile), which also searches the queries it flags
  // once per device (function attributes belong to the device the context is on, not to the process): the pipelines'
  // dynamic shared memory, the whole shared-memory carveout, and how many blocks of each pass are resident per SM
  // ([0] / [1]: cached pass p2p / combined, [2] / [3]: cold pass)
  static bool attr_set_dev[64] = {};
  static int resident_dev[64][4] = {};
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
    CB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident[2], icp_search_kernel<kModeP2PCentered>, kBlock, 0));
    CB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident[3], icp_search_kernel<kModeCombined>, kBlock, 0));
    attr_set = true;
  }
  // persistent passes: a whole number of resident blocks per SM (never more blocks than tiles / chunks need)
  const bool p2p = prm->metric == CB_ICP_POINT_TO_POINT;
  const int per_sm = std::max(1, resident[p2p ? 0 : 1]);
  const size_t tile = (size_t)pipe_qpt(!p2p) * kBlock;
  const int blocks_cached = grid_for(ctx, ns, tile, per_sm);
  const int blocks_cold = grid_for(ctx, ns, kBlock, std::max(1, resident[p2p ? 2 : 3]));
  // the cached pass's flagged-query lists: per warp, room for every query of its block's tiles (about n_src in all)
  const size_t per_warp = ((ns + tile - 1) / tile + blocks_cached - 1) / blocks_cached * (tile / (kBlock / 32));
  const size_t flagged_need = per_warp * (size_t)blocks_cached * (kBlock / 32);
  const bool projective = icp->proj.on;
  const int blocks_proj = grid_for(ctx, ns, kBlock, proj_min_blocks(!p2p));
  if (projective) {
    a.proj_map = icp->proj.d_map;
    a.prj = icp->proj.prj;
  } else if (icp->loop_flagged_cap < flagged_need) {
    if (icp->d_loop_flagged) CB_TRY(icp->mem.free(icp->d_loop_flagged));
    icp->d_loop_flagged = nullptr;
    icp->loop_flagged_cap = 0;
    CB_TRY(icp->mem.alloc(&icp->d_loop_flagged, flagged_need));
    icp->loop_flagged_cap = flagged_need;
  }
  a.flagged = icp->d_loop_flagged;
  a.flagged_per_warp = (uint32_t)per_warp;
  CB_TRY(get_reduce_scratch(ctx, std::max(std::max(blocks_cold, blocks_cached), blocks_proj), kMaxValues, &a.rs));
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
        CB_TRY(enqueue_iteration<kModeP2PCentered>(ctx, a, issued + k, blocks_cold, blocks_cached, blocks_proj));
      else
        CB_TRY(enqueue_iteration<kModeCombined>(ctx, a, issued + k, blocks_cold, blocks_cached, blocks_proj));
      if (timing) CB_CUDA(cudaEventRecord(icp->events[2 * (issued + k) + 1], ctx->stream));
    }
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
  icp->loop_last = !projective;  // (cb_icp_loop_cache inspects the kd-tree search's cache)
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
