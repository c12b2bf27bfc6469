// Mean-shift clustering (product code, sm_90a).
// Replaces MeanShift<float, 3>::cluster (clustering/mean_shift.hpp:37-115, :118-124). DESIGN §4.11 pins the semantics.
//
// Shift loop, host-driven: one host read per iteration of the per-seed list sizes (to cut the active seeds into
// batches of at most a pair budget) and one of the number of seeds still active. Per batch the radius lists of
// radius_lists.cuh (count -> scan -> fill -> (d2, index) heap sort) feed shift_kernel, which sums every list in
// that order with the reference's fp32 operations (no FMA, 1 / W then three multiplies), applies the convergence
// test, writes the seed back and compacts the ids of the seeds still active.
//
// Clustering, exact and parallel. Clusters are created in seed order, so seed i starts a cluster (is a
// representative) iff no representative j < i lies within cluster_tol, and its label is the representative with the
// smallest index within cluster_tol: the lexicographically first independent set of the tol-graph. Rounds over a
// grid built on the shifted seeds decide it: a seed becomes a non-representative once a lower-index neighbour is a
// representative, and a representative once all its lower-index neighbours are non-representatives. The decisions
// are monotone and each is valid whatever mix of old and new states a thread observes, so the result does not depend
// on scheduling. Non-finite seeds (and every seed when !(cluster_tol^2 > 0)) are singletons. Clusters are numbered
// by representative index; a stable radix sort of (cluster, seed) gives the CSR; one thread per cluster sums its
// mode serially in seed order (the reference's order), so that pass costs as much as the largest cluster.
#include "cb_internal.hpp"
#include "grid_sweep.cuh"
#include "launch.cuh"
#include "radius_lists.cuh"
#include <algorithm>
#include <cstdlib>
#include <vector>

using namespace cb;

namespace {

constexpr int kBlock = 128;
constexpr uint32_t kUndecided = 0, kRep = 1, kNonRep = 2;
// The clustering sweeps are launched with at most 8 blocks per SM; saying so lets ptxas keep the sweep state in
// registers (left to itself it aims higher, at 32 registers, and spills).
constexpr int kSweepBlocksPerSm = 8;

// packed xyz -> float4 seeds; active ids 0..n-1
__global__ void init_seeds_kernel(const float* __restrict__ xyz, uint32_t n, float4* __restrict__ seeds,
                                  uint32_t* __restrict__ active) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    seeds[i] = make_float4(xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2], 0.f);
    active[i] = i;
  }
}

// radius-list queries of the active seeds: q[a] = (seed[active[a]], slot a)
__global__ void queries_kernel(const float4* __restrict__ seeds, const uint32_t* __restrict__ active, uint32_t n,
                               float4* __restrict__ q) {
  for (uint32_t a = blockIdx.x * blockDim.x + threadIdx.x; a < n; a += gridDim.x * blockDim.x) {
    const float4 s = seeds[active[a]];
    q[a] = make_float4(s.x, s.y, s.z, __int_as_float((int)a));
  }
}

// One active seed per thread (mean_shift.hpp:59-76). off/idx/d2: the batch's lists, ascending (d2, index).
__global__ void shift_kernel(const float* __restrict__ raw, const uint32_t* __restrict__ active, uint32_t nb,
                             const uint32_t* __restrict__ off, const int* __restrict__ idx, const float* __restrict__ d2,
                             int rbf, float coeff, float tol2, float4* __restrict__ seeds, uint32_t* __restrict__ next,
                             uint32_t* next_count) {
  for (uint32_t a = blockIdx.x * blockDim.x + threadIdx.x; a < nb; a += gridDim.x * blockDim.x) {
    const uint32_t id = active[a];
    const uint32_t b = off[a], e = off[a + 1];
    float ax = 0.f, ay = 0.f, az = 0.f, w_sum = 0.f;
    for (uint32_t j = b; j < e; ++j) {
      const size_t p = 3 * (size_t)idx[j];
      const float w = rbf ? expf(__fmul_rn(coeff, d2[j])) : 1.0f;
      ax = __fadd_rn(ax, __fmul_rn(w, __ldg(raw + p)));
      ay = __fadd_rn(ay, __fmul_rn(w, __ldg(raw + p + 1)));
      az = __fadd_rn(az, __fmul_rn(w, __ldg(raw + p + 2)));
      w_sum = __fadd_rn(w_sum, w);
    }
    const float inv = __fdiv_rn(1.0f, w_sum);
    const float mx = __fmul_rn(ax, inv), my = __fmul_rn(ay, inv), mz = __fmul_rn(az, inv);
    const float4 s = seeds[id];
    const float r = rule::contract_d2(s.x, s.y, s.z, mx, my, mz);
    seeds[id] = make_float4(mx, my, mz, 0.f);
    if (!(r < tol2)) next[atomicAdd(next_count, 1u)] = id;
  }
}

// shifted seeds -> packed xyz (the clustering grid's input and the host output)
__global__ void pack_kernel(const float4* __restrict__ seeds, uint32_t n, float* __restrict__ xyz) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 s = seeds[i];
    xyz[3 * (size_t)i] = s.x;
    xyz[3 * (size_t)i + 1] = s.y;
    xyz[3 * (size_t)i + 2] = s.z;
  }
}

// ---- deduplication of exactly coincident seeds ----
// Seeds are sorted on their coordinate bits (stable: z, then (x, y)), so every group of bit-identical seeds is a run in
// ascending seed order and its first element is its lowest-index member. With cluster_tol^2 > 0 every other member
// lies at distance 0 from it: it is never a representative (its lower-index twin is a representative or has one
// within cluster_tol) and its label is the twin's. So only the first member of each group (its head) takes part in
// the clustering sweeps; a cluster of a million bit-identical seeds costs one sweep, not a million squared tests.
// Non-finite seeds are groups of their own (singletons, inert in the grid).
__global__ void key_z_kernel(const float4* __restrict__ seeds, uint32_t n, uint64_t* __restrict__ keys,
                             uint32_t* __restrict__ vals) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    keys[i] = (uint32_t)__float_as_uint(seeds[i].z);
    vals[i] = i;
  }
}

__global__ void key_xy_kernel(const float4* __restrict__ seeds, const uint32_t* __restrict__ vals, uint32_t n,
                              uint64_t* __restrict__ keys) {
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const float4 s = seeds[vals[k]];
    keys[k] = ((uint64_t)__float_as_uint(s.x) << 32) | __float_as_uint(s.y);
  }
}

__device__ __forceinline__ bool group_start(const float4* __restrict__ seeds, const uint32_t* __restrict__ vals,
                                            uint32_t k) {
  const float4 s = seeds[vals[k]];
  if (k == 0 || !finite_point(s.x, s.y, s.z)) return true;
  const float4 t = seeds[vals[k - 1]];
  return __float_as_uint(s.x) != __float_as_uint(t.x) || __float_as_uint(s.y) != __float_as_uint(t.y) ||
         __float_as_uint(s.z) != __float_as_uint(t.z);
}

__global__ void start_kernel(const float4* __restrict__ seeds, const uint32_t* __restrict__ vals, uint32_t n,
                             uint32_t* __restrict__ flag) {
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
    flag[k] = group_start(seeds, vals, k) ? 1u : 0u;
}

// gid: exclusive scan of the start flags. Group g's head id, its packed xyz (the grid's input: grid point g is
// group g) and every seed's group.
__global__ void group_kernel(const float4* __restrict__ seeds, const uint32_t* __restrict__ vals,
                             const uint32_t* __restrict__ gid, uint32_t n, uint32_t* __restrict__ head,
                             float* __restrict__ head_xyz, uint32_t* __restrict__ grp) {
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const bool st = group_start(seeds, vals, k);
    const uint32_t g = gid[k] + (st ? 0u : 0xffffffffu);
    const uint32_t i = vals[k];
    grp[i] = g;
    if (st) {
      const float4 s = seeds[i];
      head[g] = i;
      head_xyz[3 * (size_t)g] = s.x;
      head_xyz[3 * (size_t)g + 1] = s.y;
      head_xyz[3 * (size_t)g + 2] = s.z;
    }
  }
}

// non-finite heads are representatives from the start
__global__ void state_init_kernel(const float* __restrict__ head_xyz, uint32_t ng, uint32_t* __restrict__ state) {
  for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += gridDim.x * blockDim.x) {
    const float* h = head_xyz + 3 * (size_t)g;
    state[g] = finite_point(h[0], h[1], h[2]) ? kUndecided : kRep;
  }
}

// One round of the representative decision over the grid of group heads: grid point q is group q, at head_xyz[q],
// with seed id head[q]; state is indexed by group.
__global__ void __launch_bounds__(kBlock, kSweepBlocksPerSm) round_kernel(const GridView g, const float* __restrict__ head_xyz,
                                                                          const uint32_t* __restrict__ head, uint32_t ng,
                                                                          float tol2, uint32_t* state, uint32_t* undecided) {
  volatile uint32_t* st = state;
  for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < ng; q += gridDim.x * blockDim.x) {
    if (st[q] != kUndecided) continue;
    const uint32_t i = __ldg(head + q);
    const float sx = __ldg(head_xyz + 3 * (size_t)q), sy = __ldg(head_xyz + 3 * (size_t)q + 1),
                sz = __ldg(head_xyz + 3 * (size_t)q + 2);
    bool rep_below = false, pending = false;
    grid_sweep(
        g, sx, sy, sz, [&]() { return tol2; },
        [&](uint32_t b, uint32_t e) {
          for (uint32_t j = b; j < e; ++j) {
            const float4 p = __ldg(g.pts + j);
            const uint32_t o = (uint32_t)__float_as_int(p.w);
            if (__ldg(head + o) >= i || !(rule::contract_d2(sx, sy, sz, p.x, p.y, p.z) < tol2)) continue;
            const uint32_t v = st[o];
            rep_below |= v == kRep;
            pending |= v == kUndecided;
          }
        },
        [&]() { rep_below = pending = false; }, 0u);
    if (rep_below)
      st[q] = kNonRep;
    else if (!pending)
      st[q] = kRep;
    else
      atomicAdd(undecided, 1u);
  }
}

// representative of every group (seed id of the smallest-index representative head within tol2; the head itself for
// a representative)
__global__ void __launch_bounds__(kBlock, kSweepBlocksPerSm) rep_kernel(const GridView g, const float* __restrict__ head_xyz,
                                                                        const uint32_t* __restrict__ head, uint32_t ng,
                                                                        float tol2, const uint32_t* __restrict__ state,
                                                                        uint32_t* __restrict__ rep_id) {
  for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < ng; q += gridDim.x * blockDim.x) {
    const uint32_t i = head[q];
    if (state[q] == kRep) {
      rep_id[q] = i;
      continue;
    }
    const float sx = head_xyz[3 * (size_t)q], sy = head_xyz[3 * (size_t)q + 1], sz = head_xyz[3 * (size_t)q + 2];
    uint32_t best = i;
    grid_sweep(
        g, sx, sy, sz, [&]() { return tol2; },
        [&](uint32_t b, uint32_t e) {
          for (uint32_t j = b; j < e; ++j) {
            const float4 p = __ldg(g.pts + j);
            const uint32_t o = (uint32_t)__float_as_int(p.w);
            const uint32_t h = head[o];
            if (h < best && state[o] == kRep && rule::contract_d2(sx, sy, sz, p.x, p.y, p.z) < tol2) best = h;
          }
        },
        [&]() { best = i; }, 0u);
    rep_id[q] = best;
  }
}

// every seed's representative (its group's) and the representative flags of the cluster numbering scan; grp == NULL:
// every seed is a singleton
__global__ void seed_rep_kernel(const uint32_t* __restrict__ grp, const uint32_t* __restrict__ rep_id, uint32_t n,
                                uint32_t* __restrict__ rep_of, uint32_t* __restrict__ flag) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t r = grp ? rep_id[grp[i]] : i;
    rep_of[i] = r;
    flag[i] = r == i ? 1u : 0u;
  }
}

// cluster of every seed, the cluster sizes and the (cluster, seed) pairs of the CSR sort
__global__ void cluster_kernel(const uint32_t* __restrict__ rep_of, const uint32_t* __restrict__ cid, uint32_t n,
                               uint32_t* size, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t c = cid[rep_of[i]];
    atomicAdd(size + c, 1u);
    keys[i] = c;
    vals[i] = i;
  }
}

// mean_shift.hpp:104-112: one thread per cluster, members in ascending seed order
__global__ void modes_kernel(const float4* __restrict__ seeds, const uint32_t* __restrict__ off,
                             const uint32_t* __restrict__ members, uint32_t m, float* __restrict__ modes) {
  for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < m; c += gridDim.x * blockDim.x) {
    const uint32_t b = off[c], e = off[c + 1];
    float x = 0.f, y = 0.f, z = 0.f;
    for (uint32_t j = b; j < e; ++j) {
      const float4 s = seeds[members[j]];
      x = __fadd_rn(x, s.x);
      y = __fadd_rn(y, s.y);
      z = __fadd_rn(z, s.z);
    }
    const float inv = __fdiv_rn(1.0f, __uint2float_rn(e - b));
    modes[3 * (size_t)c] = __fmul_rn(x, inv);
    modes[3 * (size_t)c + 1] = __fmul_rn(y, inv);
    modes[3 * (size_t)c + 2] = __fmul_rn(z, inv);
  }
}

int bits_for(uint64_t v) {
  int b = 0;
  while (b < 64 && (v >> b) != 0) ++b;
  return b;
}

// Pairs per batch of the shift loop (2^28 by default: 2 GiB of lists). CB_MEAN_SHIFT_PAIR_BUDGET overrides it, e.g.
// to force many batches; a batch never exceeds 2^32 - 1 pairs (the lists use 32-bit offsets).
uint64_t pair_budget() {
  uint64_t b = 1ull << 28;
  if (const char* s = std::getenv("CB_MEAN_SHIFT_PAIR_BUDGET")) {
    const unsigned long long v = std::strtoull(s, nullptr, 10);
    if (v > 0) b = v;
  }
  return std::min<uint64_t>(b, 0xffffffffull);
}


}  // namespace

extern "C" int cb_cloud_mean_shift(cb_context* ctx, cb_cloud* cloud, const cb_mean_shift_params* prm,
                                   const float* seeds, size_t n_seeds, float* shifted_seeds, uint64_t* point_to_cluster,
                                   uint64_t* cluster_offsets, uint64_t* cluster_points, float* modes,
                                   size_t* num_clusters, uint64_t* iterations, float* gpu_ms,
                                   float* gpu_ms_shift) {
  CB_CHECK(ctx && cloud && prm && num_clusters && iterations, CB_ERR_INVALID, "null argument");
  CB_CHECK(cloud->ctx == ctx, CB_ERR_INVALID, "cloud belongs to another context");
  CB_CHECK(cloud->index_offset == 0, CB_ERR_UNSUPPORTED, "mean-shift is single-GPU: the cloud must have index_offset 0");
  CB_CHECK(prm->weight_kind == CB_WEIGHT_UNITY || prm->weight_kind == CB_WEIGHT_RBF, CB_ERR_INVALID,
           "unknown weight kind");
  if (!seeds) n_seeds = cloud->n;
  CB_CHECK(n_seeds < (1ull << 31), CB_ERR_UNSUPPORTED, "more than 2^31 - 1 seeds");
  CB_CHECK(n_seeds == 0 || cloud->n > 0, CB_ERR_INVALID, "mean-shift over an empty cloud");
  CB_CHECK(n_seeds == 0 || (shifted_seeds && point_to_cluster && cluster_offsets && cluster_points && modes),
           CB_ERR_INVALID, "null output array");
  CB_CUDA(cudaSetDevice(ctx->device));
  if (gpu_ms) *gpu_ms = 0.f;
  if (gpu_ms_shift) *gpu_ms_shift = 0.f;
  *num_clusters = 0;
  *iterations = 0;
  if (cluster_offsets) cluster_offsets[0] = 0;
  const uint64_t max_iter = prm->max_iter;
  if (n_seeds == 0) {
    *iterations = max_iter > 0 ? 1 : 0;  // the loop runs once over no seeds and finds them all converged
    return CB_OK;
  }
  CB_TRY(ensure_index(cloud));
  const uint32_t ns = (uint32_t)n_seeds;
  const float r2 = prm->kernel_radius * prm->kernel_radius;
  const float tol2 = prm->convergence_tol * prm->convergence_tol;
  const float ctol2 = prm->cluster_tol * prm->cluster_tol;
  const int rbf = prm->weight_kind == CB_WEIGHT_RBF;
  const uint64_t budget = pair_budget();

  DeviceScope scope(ctx);
  float4 *d_seeds, *d_q;
  uint32_t *d_act, *d_next, *d_cnt, *d_off, *d_counter;
  float* d_xyz;
  CB_TRY(scope.alloc(&d_seeds, ns));
  CB_TRY(scope.alloc(&d_q, ns));
  CB_TRY(scope.alloc(&d_act, ns));
  CB_TRY(scope.alloc(&d_next, ns));
  CB_TRY(scope.alloc(&d_cnt, ns));
  CB_TRY(scope.alloc(&d_off, (size_t)ns + 1));
  CB_TRY(scope.alloc(&d_counter, 1));
  CB_TRY(scope.alloc(&d_xyz, 3 * (size_t)ns));
  const int eb = grid_for(ctx, ns, 256);

  ScopedEvents ev, ev2;  // ev2.e0: end of the shift loop
  if (gpu_ms || gpu_ms_shift) {
    CB_TRY(ev.create());
    CB_TRY(ev2.create());
    CB_CUDA(cudaEventRecord(ev.e0, ctx->stream));
  }
  if (seeds) {
    CB_CUDA(cudaMemcpyAsync(d_xyz, seeds, 3 * (size_t)ns * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  }
  CB_TRY(launch(ctx, init_seeds_kernel, eb, 256, 0, seeds ? d_xyz : cloud->d_raw, ns, d_seeds, d_act));

  // ---- shift (mean_shift.hpp:55-82) ----
  const GridView g = grid_view(cloud);
  const Rigid I = rigid_from_t12(nullptr);
  std::vector<uint32_t> h_cnt;
  int* d_idx = nullptr;
  float* d_d2 = nullptr;
  uint64_t pair_cap = 0;
  uint32_t n_act = ns;
  uint64_t iters = 0;
  while (iters < max_iter) {
    CB_CUDA(cudaMemsetAsync(d_counter, 0, sizeof(uint32_t), ctx->stream));
    CB_TRY(launch(ctx, queries_kernel, grid_for(ctx, n_act, 256), 256, 0, d_seeds, d_act, n_act, d_q));
    // list sizes of every active seed (r2 <= 0 or NaN: every list is empty, nothing to search)
    if (r2 > 0.f) {
      CB_TRY(launch(ctx, radius_kernel<false>, grid_for(ctx, n_act, kRadiusBlock), kRadiusBlock, 0, g, d_q, n_act, I,
                    r2, d_cnt, nullptr, nullptr, nullptr));
    } else {
      CB_CUDA(cudaMemsetAsync(d_cnt, 0, n_act * sizeof(uint32_t), ctx->stream));
    }
    h_cnt.resize(n_act);
    CB_CUDA(cudaMemcpyAsync(h_cnt.data(), d_cnt, n_act * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    // batches of consecutive active seeds holding at most `budget` pairs (a seed whose list alone exceeds it gets a
    // batch of its own: lists hold fewer than 2^31 entries)
    for (uint32_t b0 = 0; b0 < n_act;) {
      uint64_t pairs = h_cnt[b0];
      uint32_t b1 = b0 + 1;
      while (b1 < n_act && pairs + h_cnt[b1] <= budget) pairs += h_cnt[b1++];
      const uint32_t nb = b1 - b0;
      if (pairs > pair_cap) {
        CB_TRY(scope.free(d_idx));
        CB_TRY(scope.free(d_d2));
        pair_cap = std::max<uint64_t>(pairs, std::min<uint64_t>(budget, 2 * pair_cap));
        CB_TRY(scope.alloc(&d_idx, pair_cap));
        CB_TRY(scope.alloc(&d_d2, pair_cap));
      }
      // the batch's offsets live in d_off[b0 .. b1] (radius_kernel indexes them by the query's slot, b0 + i)
      uint32_t* off = d_off + b0;
      CB_CUDA(cudaMemcpyAsync(off, d_cnt + b0, nb * sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->stream));
      CB_TRY(exclusive_scan_u32(ctx, off, nb, (uint32_t)pairs));
      const int qb = grid_for(ctx, nb, kRadiusBlock);
      if (pairs > 0) {
        CB_TRY(launch(ctx, radius_kernel<true>, qb, kRadiusBlock, 0, g, d_q + b0, nb, I, r2, nullptr, d_off, d_idx,
                      d_d2));
        CB_TRY(launch(ctx, segment_heapsort_kernel, qb, kRadiusBlock, 0, off, nb, d_idx, d_d2));
      }
      CB_TRY(launch(ctx, shift_kernel, grid_for(ctx, nb, kBlock), kBlock, 0, cloud->d_raw, d_act + b0, nb, off, d_idx,
                    d_d2, rbf, prm->weight_coeff, tol2, d_seeds, d_next, d_counter));
      b0 = b1;
    }
    CB_CUDA(cudaMemcpyAsync(&n_act, d_counter, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    std::swap(d_act, d_next);
    ++iters;
    if (n_act == 0) break;
  }

  // ---- cluster (mean_shift.hpp:84-100) ----
  if (ev2.e0) CB_CUDA(cudaEventRecord(ev2.e0, ctx->stream));
  CB_TRY(launch(ctx, pack_kernel, eb, 256, 0, d_seeds, ns, d_xyz));
  uint32_t *d_rep, *d_flag;
  CB_TRY(scope.alloc(&d_rep, ns));
  CB_TRY(scope.alloc(&d_flag, (size_t)ns + 1));
  uint64_t *d_keys, *d_keys_tmp;
  uint32_t *d_vals, *d_vals_tmp;
  CB_TRY(scope.alloc(&d_keys, ns));
  CB_TRY(scope.alloc(&d_keys_tmp, ns));
  CB_TRY(scope.alloc(&d_vals, ns));
  CB_TRY(scope.alloc(&d_vals_tmp, ns));
  if (!(ctol2 > 0.f)) {  // every seed is a singleton
    CB_TRY(launch(ctx, seed_rep_kernel, eb, 256, 0, nullptr, nullptr, ns, d_rep, d_flag));
  } else {
    // groups of bit-identical seeds (see key_z_kernel)
    uint32_t *d_head, *d_grp, *d_state, *d_rep_id;
    float* d_hxyz;
    CB_TRY(scope.alloc(&d_head, ns));
    CB_TRY(scope.alloc(&d_grp, ns));
    CB_TRY(scope.alloc(&d_hxyz, 3 * (size_t)ns));
    CB_TRY(launch(ctx, key_z_kernel, eb, 256, 0, d_seeds, ns, d_keys, d_vals));
    CB_TRY(radix_sort_pairs_u64(ctx, d_keys, d_vals, d_keys_tmp, d_vals_tmp, ns, 32));
    CB_TRY(launch(ctx, key_xy_kernel, eb, 256, 0, d_seeds, d_vals, ns, d_keys));
    CB_TRY(radix_sort_pairs_u64(ctx, d_keys, d_vals, d_keys_tmp, d_vals_tmp, ns, 64));
    CB_TRY(launch(ctx, start_kernel, eb, 256, 0, d_seeds, d_vals, ns, d_flag));
    uint32_t last_start = 0, ng = 0;
    CB_CUDA(cudaMemcpyAsync(&last_start, d_flag + ns - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CB_TRY(exclusive_scan_u32(ctx, d_flag, ns, 0u));
    CB_CUDA(cudaMemcpyAsync(&ng, d_flag + ns - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CB_TRY(launch(ctx, group_kernel, eb, 256, 0, d_seeds, d_vals, d_flag, ns, d_head, d_hxyz, d_grp));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    ng += last_start;
    CB_TRY(scope.alloc(&d_state, ng));
    CB_TRY(scope.alloc(&d_rep_id, ng));
    const int gb = grid_for(ctx, ng, 256);
    CB_TRY(launch(ctx, state_init_kernel, gb, 256, 0, d_hxyz, ng, d_state));
    cb_cloud* sc = nullptr;  // grid over the group heads (non-finite ones are inert in it)
    CB_TRY(cb_cloud_create_from_device(ctx, d_hxyz, nullptr, ng, 0, &sc));
    struct CloudGuard {
      cb_cloud* c;
      ~CloudGuard() { cb_cloud_destroy(c); }
    } guard{sc};
    CB_TRY(ensure_index(sc));
    const GridView sg = grid_view(sc);
    const int rb = grid_for(ctx, ng, kBlock);
    for (;;) {
      CB_CUDA(cudaMemsetAsync(d_counter, 0, sizeof(uint32_t), ctx->stream));
      CB_TRY(launch(ctx, round_kernel, rb, kBlock, 0, sg, d_hxyz, d_head, ng, ctol2, d_state, d_counter));
      uint32_t undecided = 0;
      CB_CUDA(cudaMemcpyAsync(&undecided, d_counter, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
      CB_CUDA(cudaStreamSynchronize(ctx->stream));
      if (undecided == 0) break;
    }
    CB_TRY(launch(ctx, rep_kernel, rb, kBlock, 0, sg, d_hxyz, d_head, ng, ctol2, d_state, d_rep_id));
    CB_TRY(launch(ctx, seed_rep_kernel, eb, 256, 0, d_grp, d_rep_id, ns, d_rep, d_flag));
  }
  // clusters numbered by representative index
  uint32_t last_flag = 0;
  CB_CUDA(cudaMemcpyAsync(&last_flag, d_flag + ns - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CB_TRY(exclusive_scan_u32(ctx, d_flag, ns, 0u));
  uint32_t m = 0;
  CB_CUDA(cudaMemcpyAsync(&m, d_flag + ns - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  m += last_flag;  // exclusive scan: the count is the last prefix plus the last flag

  uint32_t* d_size;
  float* d_modes;
  CB_TRY(scope.alloc(&d_size, (size_t)m + 1));
  CB_TRY(scope.alloc(&d_modes, 3 * (size_t)m));
  CB_CUDA(cudaMemsetAsync(d_size, 0, ((size_t)m + 1) * sizeof(uint32_t), ctx->stream));
  CB_TRY(launch(ctx, cluster_kernel, eb, 256, 0, d_rep, d_flag, ns, d_size, d_keys, d_vals));
  // cluster -> seeds: stable sort of (cluster, seed) in seed order
  CB_TRY(radix_sort_pairs_u64(ctx, d_keys, d_vals, d_keys_tmp, d_vals_tmp, ns, bits_for(m)));
  CB_TRY(exclusive_scan_u32(ctx, d_size, m, ns));
  CB_TRY(launch(ctx, modes_kernel, grid_for(ctx, m, kBlock), kBlock, 0, d_seeds, d_size, d_vals, m, d_modes));
  if (ev.e1) CB_CUDA(cudaEventRecord(ev.e1, ctx->stream));

  std::vector<uint32_t> h_pts(ns), h_off((size_t)m + 1);
  CB_CUDA(cudaMemcpyAsync(shifted_seeds, d_xyz, 3 * (size_t)ns * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaMemcpyAsync(modes, d_modes, 3 * (size_t)m * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaMemcpyAsync(h_off.data(), d_size, ((size_t)m + 1) * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaMemcpyAsync(h_pts.data(), d_vals, ns * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  if (gpu_ms) CB_CUDA(cudaEventElapsedTime(gpu_ms, ev.e0, ev.e1));
  if (gpu_ms_shift) CB_CUDA(cudaEventElapsedTime(gpu_ms_shift, ev.e0, ev2.e0));
  for (uint32_t c = 0; c <= m; c++) cluster_offsets[c] = h_off[c];
  for (uint32_t c = 0; c < m; c++)
    for (uint32_t j = h_off[c]; j < h_off[c + 1]; j++) point_to_cluster[h_pts[j]] = c;
  for (uint32_t i = 0; i < ns; i++) cluster_points[i] = h_pts[i];
  *num_clusters = m;
  *iterations = iters;
  return CB_OK;
}
