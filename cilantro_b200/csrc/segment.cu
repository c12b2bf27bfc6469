// Connected-component extraction (product code, sm_90a).
// Replaces extractConnectedComponents / ConnectedComponentExtraction3f::segment (clustering/
// connected_component_extraction.hpp:163-265, :368-428) over a cloud's own neighbourhoods. DESIGN §4.10 pins the
// semantics: directed edges p -> q for q at position >= 1 of N(p) (ascending (d2, original index)) that pass the
// evaluator; labelled set = points reachable from the seeds; segments = weakly connected components of the labelled
// points; size filter; order by size descending, ties by the smallest seed position.
//
// Union-find over 32-bit parents indexed by original point index. A hook links the larger root under the smaller
// one with atomicCAS (retried when the CAS loses a race); finds halve paths with plain stores (a store only ever
// writes an ancestor, and parents only decrease). The partition does not depend on launch or atomic order, and the
// root of every component is its smallest index.
//   all seeds: one thread per point (cell-sorted order) runs the neighbourhood sweep and unions along every
//              accepted out-edge (radius: every accepted pair q > p, see below); no edge list is materialised, so
//              radius neighbourhoods stay unbounded.
//   seed list: a level-synchronous BFS; every expanded point runs the same sweep, unions along its accepted edges
//              and claims unvisited targets for the next frontier. Visited = labelled.
// Then: sizes per root, the min / max filter, a radix sort of the kept segments on (size desc, tie key asc), the
// point -> cluster scatter and a stable radix sort of (cluster, point) pairs for the cluster -> points lists.
#include "cb_internal.hpp"
#include "grid_sweep.cuh"
#include "kbest.cuh"
#include "launch.cuh"
#include "similarity_rule.hpp"
#include <algorithm>
#include <cmath>
#include <vector>

using namespace cb;

namespace {

constexpr int kBlock = 128;
constexpr uint32_t kNone = 0xffffffffu;

// Event counts of the union-find for diagnostics. Only a build with -DCB_SEGMENT_COUNTERS=1 reads them
// (tools/segment_counters.py); otherwise the increments are dead code and compile away.
struct UfStats {
  uint32_t unions = 0, find_steps = 0, cas = 0, cas_failed = 0, resets = 0;
};

__device__ __forceinline__ uint32_t uf_find(uint32_t* parent, uint32_t x, UfStats& st) {
  volatile uint32_t* p = parent;
  for (;;) {
    const uint32_t px = p[x];
    ++st.find_steps;
    if (px == x) return x;
    const uint32_t gp = p[px];
    if (gp != px) p[x] = gp;  // path halving
    x = gp;
  }
}

__device__ __forceinline__ void uf_union(uint32_t* parent, uint32_t a, uint32_t b, UfStats& st) {
  ++st.unions;
  for (;;) {
    a = uf_find(parent, a, st);
    b = uf_find(parent, b, st);
    if (a == b) return;
    const uint32_t hi = max(a, b), lo = min(a, b);
    ++st.cas;
    if (atomicCAS(parent + hi, hi, lo) == hi) return;
    ++st.cas_failed;
    // hi was hooked by another thread meanwhile: retry from the current roots
  }
}

struct SegArgs {
  GridView g;
  sim::Rule rule;
  const float4* nrm;      // cell order (kNormals) or nullptr
  const float4* col;      // cell order (kColors) or nullptr
  const uint32_t* rank;   // original index -> cell position
  uint32_t* parent;       // n, original order
  int k;                  // 0: radius neighbourhood (d2 < r2); > 0: the k nearest with d2 < r2
  float r2;
  // seeded BFS only
  const uint32_t* frontier;
  uint32_t nfront;
  uint32_t* visited;      // n flags, original order
  uint32_t* next;
  uint32_t* next_count;
};

#ifdef CB_SEGMENT_COUNTERS
__device__ unsigned long long g_uf_counts[5];  // unions, find steps, CAS, failed CAS, far-path resets
#endif

// One query: every out-edge of the point at cell position qpos that passes the rule is handed to emit(target).
// Launched with kBlocksPerSm blocks per SM (launch_sweep); saying so to ptxas lets it keep every loop variable in
// registers (without the hint it aims at 12 resident blocks, 40 registers, and spills the query index and the row
// budget of grid_sweep).
constexpr int kBlocksPerSm = 8;
template <int K, bool kBfs>
__global__ void __launch_bounds__(kBlock, kBlocksPerSm) segment_kernel(const SegArgs a) {
  UfStats st;
  const GridView& g = a.g;
  const uint32_t nq = kBfs ? a.nfront : g.n;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t qi = blockIdx.x * blockDim.x + threadIdx.x; qi < nq; qi += stride) {
    const uint32_t qpos = kBfs ? __ldg(a.rank + a.frontier[qi]) : qi;
    const float4 s = __ldg(g.pts + qpos);
    const uint32_t po = (uint32_t)__float_as_int(s.w);
    const uint32_t terms = a.rule.terms;
    const float4 ns = (terms & sim::kNormals) ? __ldg(a.nrm + qpos) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 cs = (terms & sim::kColors) ? __ldg(a.col + qpos) : make_float4(0.f, 0.f, 0.f, 0.f);
    // the evaluators of core/common_pair_evaluators.hpp:88-259 (terms combined with AND)
    auto accept = [&](uint32_t pos, float d2) {
      if ((terms & sim::kPoints) && !(d2 < a.rule.max_d2)) return false;
      if (terms & sim::kColors) {
        const float4 c = __ldg(a.col + pos);
        if (!(sim::color_d2(cs.x, cs.y, cs.z, c.x, c.y, c.z) < a.rule.max_c2)) return false;
      }
      if (terms & sim::kNormals) {
        const float4 m = __ldg(a.nrm + pos);
        if (!sim::dot_passes(a.rule, sim::dot3(ns.x, ns.y, ns.z, m.x, m.y, m.z))) return false;
      }
      return true;
    };
    auto emit = [&](uint32_t pos, float d2, uint32_t qo) {
      if (!accept(pos, d2)) return;
      uf_union(a.parent, po, qo, st);
      if (kBfs && atomicCAS(a.visited + qo, 0u, 1u) == 0u) a.next[atomicAdd(a.next_count, 1u)] = qo;
    };
    if constexpr (K == 0 && !kBfs) {
      // Radius, all seeds: the relation is symmetric (DESIGN §4.10), so every unordered pair is united once, from its
      // lower index; a q > p is never at position 0 of N(p) (p itself, d2 = 0, precedes it), so nothing is held back.
      const float r2 = a.r2;
      grid_sweep(
          g, s.x, s.y, s.z, [&]() { return r2; },
          [&](uint32_t b, uint32_t e) {
            for (uint32_t j = b; j < e; ++j) {
              const float4 p = __ldg(g.pts + j);
              const uint32_t oi = (uint32_t)__float_as_int(p.w);
              if (oi <= po) continue;
              const float r = rule::contract_d2(s.x, s.y, s.z, p.x, p.y, p.z);
              if (r < r2) emit(j, r, oi);
            }
          },
          [&]() { ++st.resets; }, 0u);  // (the far path re-scans from scratch: unions are idempotent)
    } else if constexpr (K == 0) {
      // Radius, seed list: N(p) is unbounded, so nothing is stored. Position 0 is the (d2, index)-minimum: the running minimum
      // is held back and emitted only once a smaller candidate displaces it; every other candidate is emitted at
      // once (something smaller was already seen, so it is not at position 0).
      const float r2 = a.r2;
      bool held = false;
      float hd = 0.f;
      uint32_t hi = 0, hpos = 0;
      grid_sweep(
          g, s.x, s.y, s.z, [&]() { return r2; },
          [&](uint32_t b, uint32_t e) {
            for (uint32_t j = b; j < e; ++j) {
              const float4 p = __ldg(g.pts + j);
              const float r = rule::contract_d2(s.x, s.y, s.z, p.x, p.y, p.z);
              if (!(r < r2)) continue;
              const uint32_t oi = (uint32_t)__float_as_int(p.w);
              if (!held) {
                held = true;
                hd = r, hi = oi, hpos = j;
              } else if (r < hd || (r == hd && oi < hi)) {
                emit(hpos, hd, hi);
                hd = r, hi = oi, hpos = j;
              } else {
                emit(j, r, oi);
              }
            }
          },
          // The far-query path restarts the scan from scratch. Unions already made stay (they are real edges and
          // unions are idempotent), but the held-back candidate must go: seen again, it would compare equal to
          // itself and be emitted as an edge to position 0.
          [&]() {
            held = false;
            ++st.resets;
          },
          0u);
    } else {
      float bd[K];
      int bi[K];
      int count = 0;
      const int k = a.k;
      const float max_d2 = a.r2;
      auto bound = [&]() { return (count == k) ? bd[k - 1] : max_d2; };
      grid_sweep(
          g, s.x, s.y, s.z, bound,
          [&](uint32_t b, uint32_t e) {
            for (uint32_t j = b; j < e; ++j) {
              const float4 p = __ldg(g.pts + j);
              const float r = rule::contract_d2(s.x, s.y, s.z, p.x, p.y, p.z);
              if (r < max_d2) kbest_insert<K>(bd, bi, k, count, r, __float_as_int(p.w));
            }
          },
          [&]() {
            count = 0;
            ++st.resets;
          },
          (uint32_t)k);
      for (int j = 1; j < count; ++j) emit(__ldg(a.rank + bi[j]), bd[j], (uint32_t)bi[j]);
    }
  }
#ifdef CB_SEGMENT_COUNTERS
  atomicAdd(&g_uf_counts[0], (unsigned long long)st.unions);
  atomicAdd(&g_uf_counts[1], (unsigned long long)st.find_steps);
  atomicAdd(&g_uf_counts[2], (unsigned long long)st.cas);
  atomicAdd(&g_uf_counts[3], (unsigned long long)st.cas_failed);
  atomicAdd(&g_uf_counts[4], (unsigned long long)st.resets);
#endif
}

__global__ void iota_kernel(uint32_t* parent, uint32_t n) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) parent[i] = i;
}

__global__ void rank_kernel(const float4* __restrict__ pts, uint32_t n, uint32_t* __restrict__ rank) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    rank[__float_as_int(pts[i].w)] = i;
}

// packed xyz in original order -> float4 in cell order
__global__ void gather_kernel(const float* __restrict__ raw, const float4* __restrict__ pts, uint32_t n,
                              float4* __restrict__ out) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const size_t o = 3 * (size_t)__float_as_int(pts[i].w);
    out[i] = make_float4(raw[o], raw[o + 1], raw[o + 2], 0.f);
  }
}

// seeds: mark visited, first frontier = the distinct seeds
__global__ void seed_kernel(const uint32_t* __restrict__ seeds, uint32_t ns, uint32_t* visited, uint32_t* front,
                            uint32_t* front_count) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += gridDim.x * blockDim.x) {
    const uint32_t s = seeds[i];
    if (atomicCAS(visited + s, 0u, 1u) == 0u) front[atomicAdd(front_count, 1u)] = s;
  }
}

// root per point (kNone = unlabelled) and the size of every component at its root
__global__ void compress_kernel(uint32_t* parent, const uint32_t* __restrict__ visited, uint32_t n,
                                uint32_t* __restrict__ root, uint32_t* size) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    uint32_t r = kNone;
    if (!visited || visited[i]) {
      UfStats st;
      r = uf_find(parent, i, st);
      atomicAdd(size + r, 1u);
    }
    root[i] = r;
  }
}

// tie key with a seed list: the smallest seed-list position of any seed in the segment
__global__ void seed_tie_kernel(const uint32_t* __restrict__ seeds, uint32_t ns, const uint32_t* __restrict__ root,
                                uint32_t* tie) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += gridDim.x * blockDim.x)
    atomicMin(tie + root[seeds[i]], i);
}

// kept segments -> (key, root); key = (size descending, tie key ascending): unique per segment, so the sorted order
// does not depend on the order the slots were taken in
__global__ void segments_kernel(const uint32_t* __restrict__ root, const uint32_t* __restrict__ size,
                                const uint32_t* __restrict__ tie, uint32_t n, uint64_t min_size, uint64_t max_size,
                                uint64_t* __restrict__ keys, uint32_t* __restrict__ vals, uint32_t* count) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (root[i] != i) continue;
    const uint32_t s = size[i];
    if (s < min_size || s > max_size) continue;
    const uint32_t slot = atomicAdd(count, 1u);
    keys[slot] = ((uint64_t)(kNone - s) << 32) | (tie ? tie[i] : i);
    vals[slot] = i;
  }
}

__global__ void cluster_id_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ roots, uint32_t m,
                                  uint32_t* __restrict__ cid, uint32_t* __restrict__ sizes) {
  for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < m; c += gridDim.x * blockDim.x) {
    cid[roots[c]] = c;
    sizes[c] = kNone - (uint32_t)(keys[c] >> 32);
  }
}

// point -> cluster (m = unlabelled) and the (cluster, point) pairs of the final stable sort, in point order
__global__ void label_kernel(const uint32_t* __restrict__ root, const uint32_t* __restrict__ cid, uint32_t n,
                             uint32_t m, uint32_t* __restrict__ p2c, uint64_t* __restrict__ keys,
                             uint32_t* __restrict__ vals) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t r = root[i];
    const uint32_t c = (r == kNone || cid[r] == kNone) ? m : cid[r];
    p2c[i] = c;
    keys[i] = c;
    vals[i] = i;
  }
}

int bits_for(uint64_t v) {
  int b = 0;
  while (b < 64 && (v >> b) != 0) ++b;
  return b;
}

template <bool kBfs>
int launch_sweep(cb_context* ctx, const SegArgs& a, uint32_t nq) {
  const int k = a.k;
  auto kernel = segment_kernel<256, kBfs>;
  if (k == 0)
    kernel = segment_kernel<0, kBfs>;
  else if (k <= 4)
    kernel = segment_kernel<4, kBfs>;
  else if (k <= 16)
    kernel = segment_kernel<16, kBfs>;
  else if (k <= 32)
    kernel = segment_kernel<32, kBfs>;
  else if (k <= 64)
    kernel = segment_kernel<64, kBfs>;
  else if (k <= 128)
    kernel = segment_kernel<128, kBfs>;
  return launch(ctx, kernel, grid_for(ctx, nq, kBlock, kBlocksPerSm), kBlock, 0, a);
}

}  // namespace

extern "C" int cb_cloud_segment(cb_context* ctx, cb_cloud* cloud, const cb_segment_params* prm, const float* normals,
                                const float* colors, const uint64_t* seeds, size_t n_seeds, uint64_t* point_to_cluster,
                                uint64_t* cluster_offsets, uint64_t* cluster_points, size_t* num_clusters,
                                float* gpu_ms) {
  CB_CHECK(ctx && cloud && prm && point_to_cluster && cluster_offsets && cluster_points && num_clusters, CB_ERR_INVALID,
           "null argument");
  CB_CHECK(cloud->ctx == ctx, CB_ERR_INVALID, "cloud belongs to another context");
  CB_CHECK(cloud->index_offset == 0, CB_ERR_UNSUPPORTED, "segmentation is single-GPU: the cloud must have index_offset 0");
  CB_CHECK(prm->k >= 0 && prm->k <= kKBestMaxK, CB_ERR_UNSUPPORTED, "k must be in [0, 256] (0 = radius neighbourhood)");
  CB_CHECK(prm->k > 0 || prm->radius2 > 0.f, CB_ERR_INVALID, "need k > 0 and/or radius2 > 0");
  CB_CHECK((prm->terms & ~(CB_SEG_POINTS | CB_SEG_NORMALS | CB_SEG_COLORS)) == 0, CB_ERR_INVALID, "unknown evaluator term");
  CB_CHECK(!(prm->terms & CB_SEG_COLORS) || colors, CB_ERR_INVALID, "the colour term needs colors");
  const size_t n = cloud->n;
  CB_CHECK(n < (size_t)kNone - 1 && n <= (size_t)INT32_MAX, CB_ERR_UNSUPPORTED, "more than 2^31 - 1 points");
  for (size_t i = 0; seeds && i < n_seeds; i++) CB_CHECK(seeds[i] < n, CB_ERR_INVALID, "seed index out of range");
  CB_CUDA(cudaSetDevice(ctx->device));
  if (gpu_ms) *gpu_ms = 0.f;
  *num_clusters = 0;
  cluster_offsets[0] = 0;
  if (n == 0) return CB_OK;
  CB_TRY(ensure_index(cloud));
  CB_CHECK(!(prm->terms & CB_SEG_NORMALS) || normals || cloud->d_nrm, CB_ERR_INVALID,
           "the normals term needs normals (host array, or normals stored in the cloud)");

  SegArgs a{};
  a.g = grid_view(cloud);
  a.rule.terms = (uint32_t)prm->terms;
  a.rule.max_d2 = prm->max_distance;
  a.rule.max_c2 = prm->max_color_diff2;
  sim::derive_angle_intervals(a.rule, prm->max_angle, prm->angle_strict != 0);
  a.k = prm->k;
  a.r2 = prm->radius2 > 0.f ? prm->radius2 : 3.402823466e38f;
  const uint32_t n32 = (uint32_t)n;
  const bool seeded = seeds != nullptr;

  DeviceScope scope(ctx);
  uint32_t *d_parent, *d_rank, *d_root, *d_size, *d_tie = nullptr, *d_visited = nullptr, *d_cnt;
  CB_TRY(scope.alloc(&d_parent, n));
  CB_TRY(scope.alloc(&d_rank, n));
  CB_TRY(scope.alloc(&d_root, n));
  CB_TRY(scope.alloc(&d_size, n));
  CB_TRY(scope.alloc(&d_cnt, 2));
  float* d_host_in = nullptr;  // staging of host normals / colours (original order)
  if ((prm->terms & (CB_SEG_NORMALS | CB_SEG_COLORS)) && (normals || colors)) CB_TRY(scope.alloc(&d_host_in, 3 * n));
  float4* d_col = nullptr;
  float4* d_nrm = cloud->d_nrm;
  const int eb = grid_for(ctx, n, 256);

  ScopedEvents ev;
  if (gpu_ms) {
    CB_TRY(ev.create());
    CB_CUDA(cudaEventRecord(ev.e0, ctx->stream));
  }
#ifdef CB_SEGMENT_COUNTERS
  const unsigned long long zero[5] = {0, 0, 0, 0, 0};
  CB_CUDA(cudaMemcpyToSymbolAsync(g_uf_counts, zero, sizeof(zero), 0, cudaMemcpyHostToDevice, ctx->stream));
#endif
  CB_TRY(launch(ctx, rank_kernel, eb, 256, 0, cloud->d_pts, n32, d_rank));
  CB_TRY(launch(ctx, iota_kernel, eb, 256, 0, d_parent, n32));
  if ((prm->terms & CB_SEG_NORMALS) && normals) {
    CB_TRY(scope.alloc(&d_nrm, n));
    CB_CUDA(cudaMemcpyAsync(d_host_in, normals, 3 * n * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    CB_TRY(launch(ctx, gather_kernel, eb, 256, 0, d_host_in, cloud->d_pts, n32, d_nrm));
  }
  if (prm->terms & CB_SEG_COLORS) {
    CB_TRY(scope.alloc(&d_col, n));
    CB_CUDA(cudaMemcpyAsync(d_host_in, colors, 3 * n * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    CB_TRY(launch(ctx, gather_kernel, eb, 256, 0, d_host_in, cloud->d_pts, n32, d_col));
  }
  a.nrm = (prm->terms & CB_SEG_NORMALS) ? d_nrm : nullptr;
  a.col = d_col;
  a.rank = d_rank;
  a.parent = d_parent;

  if (!seeded) {
    CB_TRY(launch_sweep<false>(ctx, a, n32));
  } else {
    // level-synchronous BFS from the seeds; one host read of the frontier size per level
    uint32_t *d_front, *d_next;
    CB_TRY(scope.alloc(&d_visited, n));
    CB_TRY(scope.alloc(&d_front, n));
    CB_TRY(scope.alloc(&d_next, n));
    CB_TRY(scope.alloc(&d_tie, n));
    CB_CUDA(cudaMemsetAsync(d_visited, 0, n * sizeof(uint32_t), ctx->stream));
    CB_CUDA(cudaMemsetAsync(d_cnt, 0, 2 * sizeof(uint32_t), ctx->stream));
    uint32_t* d_seeds = nullptr;
    if (n_seeds) {
      CB_CHECK(n_seeds < (size_t)kNone, CB_ERR_UNSUPPORTED, "more than 2^32 - 2 seeds");
      std::vector<uint32_t> h_seeds(n_seeds);
      for (size_t i = 0; i < n_seeds; i++) h_seeds[i] = (uint32_t)seeds[i];
      CB_TRY(scope.alloc(&d_seeds, n_seeds));
      CB_CUDA(cudaMemcpyAsync(d_seeds, h_seeds.data(), n_seeds * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
      const int sb = grid_for(ctx, n_seeds, 256);
      CB_TRY(launch(ctx, seed_kernel, sb, 256, 0, d_seeds, (uint32_t)n_seeds, d_visited, d_front, d_cnt));
    }
    a.visited = d_visited;
    a.next_count = d_cnt + 1;
    uint32_t nfront = 0;
    CB_CUDA(cudaMemcpyAsync(&nfront, d_cnt, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    while (nfront > 0) {
      a.frontier = d_front;
      a.nfront = nfront;
      a.next = d_next;
      CB_CUDA(cudaMemsetAsync(d_cnt + 1, 0, sizeof(uint32_t), ctx->stream));
      CB_TRY(launch_sweep<true>(ctx, a, nfront));
      CB_CUDA(cudaMemcpyAsync(&nfront, d_cnt + 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
      CB_CUDA(cudaStreamSynchronize(ctx->stream));
      std::swap(d_front, d_next);
    }
    CB_CUDA(cudaMemsetAsync(d_tie, 0xff, n * sizeof(uint32_t), ctx->stream));
    CB_CUDA(cudaMemsetAsync(d_size, 0, n * sizeof(uint32_t), ctx->stream));
    CB_TRY(launch(ctx, compress_kernel, eb, 256, 0, d_parent, d_visited, n32, d_root, d_size));
    if (n_seeds) {
      const int sb = grid_for(ctx, n_seeds, 256);
      CB_TRY(launch(ctx, seed_tie_kernel, sb, 256, 0, d_seeds, (uint32_t)n_seeds, d_root, d_tie));
    }
  }
  if (!seeded) {
    CB_CUDA(cudaMemsetAsync(d_size, 0, n * sizeof(uint32_t), ctx->stream));
    CB_TRY(launch(ctx, compress_kernel, eb, 256, 0, d_parent, nullptr, n32, d_root, d_size));
  }

  // kept segments, sorted on (size desc, tie key asc)
  uint64_t *d_keys, *d_keys_tmp;
  uint32_t *d_vals, *d_vals_tmp, *d_cid, *d_p2c;
  CB_TRY(scope.alloc(&d_keys, n));
  CB_TRY(scope.alloc(&d_keys_tmp, n));
  CB_TRY(scope.alloc(&d_vals, n));
  CB_TRY(scope.alloc(&d_vals_tmp, n));
  CB_TRY(scope.alloc(&d_cid, n));
  CB_TRY(scope.alloc(&d_p2c, n));
  CB_CUDA(cudaMemsetAsync(d_cnt, 0, sizeof(uint32_t), ctx->stream));
  CB_TRY(launch(ctx, segments_kernel, eb, 256, 0, d_root, d_size, seeded ? d_tie : nullptr, n32,
                (uint64_t)prm->min_segment_size, (uint64_t)prm->max_segment_size, d_keys, d_vals, d_cnt));
  uint32_t m = 0;
  CB_CUDA(cudaMemcpyAsync(&m, d_cnt, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  CB_TRY(radix_sort_pairs_u64(ctx, d_keys, d_vals, d_keys_tmp, d_vals_tmp, m, 64));
  CB_CUDA(cudaMemsetAsync(d_cid, 0xff, n * sizeof(uint32_t), ctx->stream));
  uint32_t* d_sizes = d_size;  // (the per-root sizes are no longer needed: reused for the sorted segment sizes)
  if (m) {
    CB_TRY(launch(ctx, cluster_id_kernel, eb, 256, 0, d_keys, d_vals, m, d_cid, d_sizes));
  }
  CB_TRY(launch(ctx, label_kernel, eb, 256, 0, d_root, d_cid, n32, m, d_p2c, d_keys, d_vals));
  // cluster -> points: stable sort of (cluster, point) in point order; unlabelled points (key m) sort last
  CB_TRY(radix_sort_pairs_u64(ctx, d_keys, d_vals, d_keys_tmp, d_vals_tmp, n, bits_for(m)));
  if (gpu_ms) CB_CUDA(cudaEventRecord(ev.e1, ctx->stream));

  std::vector<uint32_t> h_sizes(m), h_p2c(n), h_pts(n);
  if (m) CB_CUDA(cudaMemcpyAsync(h_sizes.data(), d_sizes, m * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaMemcpyAsync(h_p2c.data(), d_p2c, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaMemcpyAsync(h_pts.data(), d_vals, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  if (gpu_ms) CB_CUDA(cudaEventElapsedTime(gpu_ms, ev.e0, ev.e1));
#ifdef CB_SEGMENT_COUNTERS
  unsigned long long cnt[5];
  CB_CUDA(cudaMemcpyFromSymbol(cnt, g_uf_counts, sizeof(cnt)));
  fprintf(stderr, "CB_SEGMENT_COUNTERS unions=%llu find_steps=%llu cas=%llu cas_failed=%llu far_resets=%llu\n", cnt[0],
          cnt[1], cnt[2], cnt[3], cnt[4]);
#endif
  uint64_t total = 0;
  for (uint32_t c = 0; c < m; c++) {
    cluster_offsets[c] = total;
    total += h_sizes[c];
  }
  cluster_offsets[m] = total;
  for (size_t i = 0; i < n; i++) point_to_cluster[i] = h_p2c[i];
  for (uint64_t i = 0; i < total; i++) cluster_points[i] = h_pts[i];
  *num_clusters = m;
  return CB_OK;
}
