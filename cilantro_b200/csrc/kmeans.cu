// k-means: fused assignment + centroid-sum kernel and the Lloyd loop (product code, sm_90a).
//
// Replaces KMeans<float,3>::cluster_ (clustering/kmeans.hpp:67-194), brute-force branch:
//   assignment  :100-119  argmin_j |c_j - p_i|^2, strict '<' scanning j ascending (lowest j wins ties)
//   update      :126-131  per-cluster sum and count (serial on the CPU)
// Arithmetic contract of the distance (oracle/cilantro_oracle.cpp): d = c - p,
//   d2 = dx*dx + (dy*dy + dz*dz), fp32 round-to-nearest, no FMA.
// Bound: FP32 pipe (8 N K flop); centroids are staged in shared memory and broadcast to the warp,
// each thread keeps kPts points in registers so one LDS.128 feeds kPts distance evaluations.
// Per-cluster sums are accumulated in double with shared-memory atomics (one block-private copy),
// then flushed with global double atomics; counts likewise.
// A point with a NaN / Inf coordinate never satisfies d < best, so it keeps label 0; it adds nothing
// to any sum or count and the empty-cluster repair never picks it (the reference leaves its label
// uninitialised and sums it, so one such point would turn centroid 0 into NaN for good).
// The Lloyd loop below runs on rows of any dimension D (KMeansData): clouds are D = 3, cb_vectors sets any D >= 1.
// D = 3 assigns with kmeans_assign_kernel, other D with kmeans_features.cu; the distance of the repair and the tol
// test is the right fold of DESIGN §4.17, which is dx*dx + (dy*dy + dz*dz) at D = 3.
#include "cb_internal.hpp"
#include "host_solve.hpp"
#include "launch.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <random>
#include <vector>

using namespace cb;

namespace {

constexpr int kBlock = 256;
#ifndef CB_KMEANS_PTS
#define CB_KMEANS_PTS 4
#endif
constexpr int kPts = CB_KMEANS_PTS;  // points per thread held in registers
constexpr int kChunk = 1024;  // centroids staged per shared-memory chunk

// sums layout in global memory: K x 4 doubles (sx, sy, sz, count)
template <bool kSmemSums>
__global__ void __launch_bounds__(kBlock) kmeans_assign_kernel(const float* __restrict__ raw, size_t n,
                                                               const float4* __restrict__ cent, int K,
                                                               uint32_t* __restrict__ labels, double* __restrict__ sums,
                                                               unsigned int* __restrict__ changed) {
  extern __shared__ unsigned char smem_raw[];
  float4* s_cent = reinterpret_cast<float4*>(smem_raw);                                   // kChunk
  double* s_sums = reinterpret_cast<double*>(smem_raw + (size_t)kChunk * sizeof(float4));  // K * 4 (if kSmemSums)
  if (kSmemSums) {
    for (int j = threadIdx.x; j < K * 4; j += kBlock) s_sums[j] = 0.0;
  }
  unsigned int any_changed = 0;
  const size_t tile = (size_t)kBlock * kPts;
  for (size_t base = (size_t)blockIdx.x * tile; base < n; base += (size_t)gridDim.x * tile) {
    float px[kPts], py[kPts], pz[kPts], best[kPts];
    int bi[kPts];
#pragma unroll
    for (int u = 0; u < kPts; u++) {
      const size_t i = base + (size_t)u * kBlock + threadIdx.x;
      const bool ok = i < n;
      px[u] = ok ? raw[3 * i] : 0.f;
      py[u] = ok ? raw[3 * i + 1] : 0.f;
      pz[u] = ok ? raw[3 * i + 2] : 0.f;
      best[u] = __int_as_float(0x7f800000);  // +inf
      bi[u] = 0;
    }
    for (int c0 = 0; c0 < K; c0 += kChunk) {
      const int cn = min(kChunk, K - c0);
      __syncthreads();
      for (int j = threadIdx.x; j < cn; j += kBlock) s_cent[j] = cent[c0 + j];
      __syncthreads();
#pragma unroll 4
      for (int j = 0; j < cn; j++) {
        const float4 c = s_cent[j];
#pragma unroll
        for (int u = 0; u < kPts; u++) {
          const float dx = __fsub_rn(c.x, px[u]), dy = __fsub_rn(c.y, py[u]), dz = __fsub_rn(c.z, pz[u]);
          const float d = __fadd_rn(__fmul_rn(dx, dx), __fadd_rn(__fmul_rn(dy, dy), __fmul_rn(dz, dz)));
          if (d < best[u]) {
            best[u] = d;
            bi[u] = c0 + j;
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < kPts; u++) {
      const size_t i = base + (size_t)u * kBlock + threadIdx.x;
      if (i < n) {
        if (labels[i] != (uint32_t)bi[u]) any_changed = 1;
        labels[i] = (uint32_t)bi[u];
        if (!(isfinite(px[u]) && isfinite(py[u]) && isfinite(pz[u]))) continue;
        double* s = (kSmemSums ? s_sums : sums) + (size_t)bi[u] * 4;
        atomicAdd(s + 0, (double)px[u]);
        atomicAdd(s + 1, (double)py[u]);
        atomicAdd(s + 2, (double)pz[u]);
        atomicAdd(s + 3, 1.0);
      }
    }
  }
  if (kSmemSums) {
    __syncthreads();
    for (int j = threadIdx.x; j < K * 4; j += kBlock) {
      const double v = s_sums[j];
      if (v != 0.0) atomicAdd(sums + j, v);
    }
  }
  if (__syncthreads_or(any_changed) && threadIdx.x == 0) atomicOr(changed, 1u);
}

// farthest member of cluster `target` from the D-vector c (kmeans.hpp:151-169) under the distance contract
// (the right fold of DESIGN §4.17; at D = 3 it is dx*dx + (dy*dy + dz*dz)): packs (dist bits, ~index)
// so that atomicMax picks the largest distance and, on ties, the LOWEST index (the serial order).
// Members with a non-finite coordinate are skipped (they are in no sum).
__global__ void farthest_member_kernel(const float* __restrict__ raw, size_t n, int D, const uint32_t* __restrict__ labels,
                                       uint32_t target, const float* __restrict__ c,
                                       unsigned long long* __restrict__ out) {
  unsigned long long best = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (labels[i] != target) continue;
    const float* p = raw + i * (size_t)D;
    bool finite = true;
    float d2 = 0.f;  // 0 + d[D-1]^2 is d[D-1]^2 exactly
    for (int j = D - 1; j >= 0; j--) {
      const float x = p[j];
      finite = finite && isfinite(x);
      const float d = __fsub_rn(c[j], x);
      d2 = __fadd_rn(__fmul_rn(d, d), d2);
    }
    if (!finite) continue;
    const unsigned long long key =
        ((unsigned long long)__float_as_uint(d2) << 32) | (unsigned long long)(0xffffffffu - (uint32_t)i);
    best = max(best, key | (1ull << 63));  // bit 63 marks "a member exists" (d >= 0 so its sign bit is free)
  }
  for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0 && best) atomicMax(out, best);
}

// the right fold of the squared difference of two D-vectors on the host (the tol test, kmeans.hpp:186-188)
float fold_d2(const float* a, const float* b, int D) {
  float acc = 0.f;
  for (int j = D - 1; j >= 0; j--) {
    const float d = a[j] - b[j];
    acc = d * d + acc;
  }
  return acc;
}

// the rows k-means runs on: a cloud's packed xyz (D = 3) or a cb_vectors set
struct KMeansData {
  const float* raw;  // n x D, point-major
  size_t n;
  int D;
};

struct KMeansBuffers {
  float* d_cent = nullptr;  // K float4 at D = 3, else K x D
  float* d_oc = nullptr;    // D: the repair's old centroid
  uint32_t* d_labels = nullptr;
  double* d_sums = nullptr;  // K x (D + 1)
  unsigned int* d_changed = nullptr;
  unsigned long long* d_far = nullptr;
};

// one assignment: labels, changed flag and the K x (D + 1) sums, downloaded to h_sums
int kmeans_step(cb_context* ctx, const KMeansData& x, const KMeansBuffers& b, const float* cent, size_t K,
                std::vector<double>& h_sums, bool* changed) {
  const size_t W = (size_t)x.D + 1;
  CB_CUDA(cudaMemsetAsync(b.d_sums, 0, K * W * sizeof(double), ctx->stream));
  CB_CUDA(cudaMemsetAsync(b.d_changed, 0, sizeof(unsigned int), ctx->stream));
  if (x.D != 3) {
    CB_CUDA(cudaMemcpyAsync(b.d_cent, cent, K * x.D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    CB_TRY(kmeans_features_assign(ctx, x.raw, x.n, x.D, b.d_cent, K, b.d_labels, b.d_sums, b.d_changed));
  } else {
    std::vector<float4> c4(K);
    for (size_t j = 0; j < K; j++) c4[j] = make_float4(cent[3 * j], cent[3 * j + 1], cent[3 * j + 2], 0.f);
    float4* d_c4 = reinterpret_cast<float4*>(b.d_cent);
    CB_CUDA(cudaMemcpyAsync(d_c4, c4.data(), K * sizeof(float4), cudaMemcpyHostToDevice, ctx->stream));
    const size_t tile = (size_t)kBlock * kPts;
    const size_t smem_sums = K * 4 * sizeof(double);
    const bool use_smem = smem_sums <= kKMeansSmemSumsBytes;
    const size_t smem = kChunk * sizeof(float4) + (use_smem ? smem_sums : 0);
    // persistent grid = SMs x resident blocks per SM (occupancy API with this launch's dynamic smem);
    // a fixed 2 blocks/SM left most warp slots empty
    auto kern = use_smem ? kmeans_assign_kernel<true> : kmeans_assign_kernel<false>;
    if (use_smem) CB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    CB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kBlock, smem));
    per_sm = std::max(1, std::min(per_sm, 6));
    CB_TRY(launch(ctx, kern, grid_for(ctx, x.n, tile, per_sm), kBlock, smem, x.raw, x.n, d_c4, (int)K, b.d_labels,
                  b.d_sums, b.d_changed));
  }
  // one all-reduce of K x 4 sums per iteration when sharded (SURVEY.md §8e; clouds only)
  if (ctx->world > 1) CB_TRY(nccl_allreduce_sum_f64(ctx, b.d_sums, K * W));
  h_sums.resize(K * W);
  unsigned int h_changed = 0;
  CB_CUDA(cudaMemcpyAsync(h_sums.data(), b.d_sums, K * W * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaMemcpyAsync(&h_changed, b.d_changed, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  if (ctx->world > 1) {
    // "any label changed on any rank": piggy-back on the (already synchronised) host flag
    double flag = h_changed ? 1.0 : 0.0;
    std::memcpy(ctx->h_result, &flag, sizeof(double));
    CB_CUDA(cudaMemcpyAsync(ctx->d_result, ctx->h_result, sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    CB_TRY(nccl_allreduce_sum_f64(ctx, ctx->d_result, 1));
    CB_CUDA(cudaMemcpyAsync(ctx->h_result, ctx->d_result, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    h_changed = ctx->h_result[0] > 0.0;
  }
  *changed = h_changed != 0;
  return CB_OK;
}

int alloc_buffers(cb_context* ctx, DeviceScope& scope, const KMeansData& x, size_t K, KMeansBuffers* b) {
  CB_TRY(scope.alloc(&b->d_cent, K * (x.D == 3 ? 4 : x.D)));
  CB_TRY(scope.alloc(&b->d_oc, (size_t)x.D));
  CB_TRY(scope.alloc(&b->d_labels, x.n));
  CB_CUDA(cudaMemsetAsync(b->d_labels, 0, std::max<size_t>(x.n, 1) * sizeof(uint32_t), ctx->stream));  // kmeans.hpp:82
  CB_TRY(scope.alloc(&b->d_sums, std::max<size_t>(K, 1) * (x.D + 1)));
  CB_TRY(scope.alloc(&b->d_changed, 1));
  CB_TRY(scope.alloc(&b->d_far, 1));
  return CB_OK;
}

int download_labels(cb_context* ctx, const KMeansBuffers& b, size_t n, uint64_t* labels) {
  if (!labels || n == 0) return CB_OK;
  std::vector<uint32_t> h(n);
  CB_CUDA(cudaMemcpyAsync(h.data(), b.d_labels, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  for (size_t i = 0; i < n; i++) labels[i] = h[i];
  return CB_OK;
}

int kmeans_assign(cb_context* ctx, const KMeansData& x, const float* centroids, size_t k, uint64_t* labels,
                  double* sums, uint64_t* counts) {
  CB_CUDA(cudaSetDevice(ctx->device));
  DeviceScope scope(ctx);
  KMeansBuffers b;
  CB_TRY(alloc_buffers(ctx, scope, x, k, &b));
  std::vector<double> h_sums;
  bool changed = false;
  CB_TRY(kmeans_step(ctx, x, b, centroids, k, h_sums, &changed));
  CB_TRY(download_labels(ctx, b, x.n, labels));
  const size_t D = x.D, W = D + 1;
  for (size_t j = 0; j < k; j++) {
    if (sums)
      for (size_t r = 0; r < D; r++) sums[D * j + r] = h_sums[W * j + r];
    if (counts) counts[j] = (uint64_t)(h_sums[W * j + D] + 0.5);
  }
  return CB_OK;
}

// the Lloyd loop of kmeans.hpp:67-194 over rows of any dimension
int kmeans_cluster(cb_context* ctx, const KMeansData& x, float* centroids, size_t k, size_t max_iter, float tol,
                   uint64_t* labels, cb_kmeans_result* res) {
  CB_CUDA(cudaSetDevice(ctx->device));
  const uint64_t launches0 = ctx->launches;
  const size_t D = x.D, W = D + 1;
  DeviceScope scope(ctx);
  KMeansBuffers b;
  CB_TRY(alloc_buffers(ctx, scope, x, k, &b));
  ScopedEvents ev;
  CB_TRY(ev.create());
  const float tol_sq = tol * tol;
  std::vector<float> old, oc(D), p(D);
  std::vector<double> s;
  size_t it = 0;
  CB_CUDA(cudaEventRecord(ev.e0, ctx->stream));
  while (it < max_iter) {
    bool changed = false;
    CB_TRY(kmeans_step(ctx, x, b, centroids, k, s, &changed));
    if (!changed && it > 0) break;                              // kmeans.hpp:122
    if (tol > 0.f) old.assign(centroids, centroids + D * k);   // :123
    // :134-176 empty-cluster repair, on the reduced sums. The farthest-member search is a device
    // reduction; in the sharded case every rank proposes its best and the global best is taken.
    std::vector<double> cnt(k);
    for (size_t j = 0; j < k; j++) cnt[j] = s[W * j + D];
    for (size_t i = 0; i < k; i++) {
      if (cnt[i] != 0.0) continue;
      size_t max_ind = 0;
      for (size_t j = 1; j < k; j++)
        if (cnt[j] > cnt[max_ind]) max_ind = j;
      // old_centroid = sum * (1 / count) in fp32 (:147-148)
      const float inv = 1.0f / (float)cnt[max_ind];
      for (size_t r = 0; r < D; r++) oc[r] = (float)s[W * max_ind + r] * inv;
      if (ctx->world > 1) {
        set_error("empty-cluster repair is not implemented for sharded k-means");
        return CB_ERR_UNSUPPORTED;
      }
      CB_CUDA(cudaMemcpyAsync(b.d_oc, oc.data(), D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
      CB_CUDA(cudaMemsetAsync(b.d_far, 0, sizeof(unsigned long long), ctx->stream));
      CB_TRY(launch(ctx, farthest_member_kernel, grid_for(ctx, x.n, 256), 256, 0, x.raw, x.n, x.D, b.d_labels,
                    (uint32_t)max_ind, b.d_oc, b.d_far));
      unsigned long long key = 0;
      CB_CUDA(cudaMemcpyAsync(&key, b.d_far, sizeof(key), cudaMemcpyDeviceToHost, ctx->stream));
      CB_CUDA(cudaStreamSynchronize(ctx->stream));
      if (!key) continue;  // cannot happen: the largest cluster has members
      const uint32_t far_idx = 0xffffffffu - (uint32_t)(key & 0xffffffffull);
      // move the point to cluster i (:172-175); note the reference does NOT add it to cluster i's sum
      const uint32_t new_label = (uint32_t)i;
      CB_CUDA(cudaMemcpyAsync(b.d_labels + far_idx, &new_label, sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
      CB_CUDA(cudaMemcpyAsync(p.data(), x.raw + D * far_idx, D * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
      CB_CUDA(cudaStreamSynchronize(ctx->stream));
      for (size_t r = 0; r < D; r++) s[W * max_ind + r] -= (double)p[r];
      cnt[max_ind] -= 1.0;
      cnt[i] += 1.0;
    }
    for (size_t j = 0; j < k; j++) {  // :179-181  centroid = sum * (1 / count)
      const float inv = 1.0f / (float)cnt[j];
      for (size_t r = 0; r < D; r++) centroids[D * j + r] = (float)s[W * j + r] * inv;
    }
    it++;
    if (tol > 0.f) {  // :186-188
      float mx = 0.f;
      for (size_t j = 0; j < k; j++) mx = std::max(mx, fold_d2(centroids + D * j, old.data() + D * j, x.D));
      if (mx < tol_sq) break;
    }
  }
  CB_CUDA(cudaEventRecord(ev.e1, ctx->stream));
  CB_TRY(download_labels(ctx, b, x.n, labels));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  float ms = 0.f;
  CB_CUDA(cudaEventElapsedTime(&ms, ev.e0, ev.e1));
  if (res) {
    res->iterations = it;
    res->gpu_ms_total = ms;
    res->kernel_launches = ctx->launches - launches0;
  }
  return CB_OK;
}

// the checks of the cb_vectors entry points: single GPU, centroid sums indexable by int
int check_vectors(cb_context* ctx, const cb_vectors* v, const float* centroids, size_t k) {
  CB_CHECK(ctx && v && centroids && k > 0, CB_ERR_INVALID, "bad arguments");
  CB_CHECK(v->ctx == ctx, CB_ERR_INVALID, "vector set belongs to another context");
  CB_CHECK(k <= (size_t)INT32_MAX / (size_t)(v->D + 1), CB_ERR_INVALID, "k x (D + 1) too large");
  CB_CHECK(ctx->world == 1, CB_ERR_UNSUPPORTED, "k-means over vector sets runs on one GPU");
  return CB_OK;
}

}  // namespace

extern "C" {

int cb_kmeans_seed_indices(size_t n, size_t k, uint32_t seed, uint64_t* out_idx) {
  CB_CHECK(out_idx && k <= n, CB_ERR_INVALID, "bad arguments");
  // KMeans::cluster(num_clusters, ...) — kmeans.hpp:38-49, seed injected for std::random_device
  std::vector<size_t> range(n);
  for (size_t i = 0; i < n; i++) range[i] = i;
  std::mt19937 rng(seed);
  size_t prev_size = n;
  for (size_t i = 0; i < k; i++) {
    std::uniform_int_distribution<size_t> dist(0, prev_size - 1);
    const size_t r = dist(rng);
    out_idx[i] = range[r];
    prev_size--;
    std::swap(range[r], range[prev_size]);
  }
  return CB_OK;
}

int cb_kmeans_assign(cb_context* ctx, const cb_cloud* pts, const float* centroids, size_t k, uint64_t* labels,
                     double* sums, uint64_t* counts) {
  CB_CHECK(ctx && pts && centroids && k > 0, CB_ERR_INVALID, "bad arguments");
  return kmeans_assign(ctx, KMeansData{pts->d_raw, pts->n, 3}, centroids, k, labels, sums, counts);
}

int cb_kmeans_cluster(cb_context* ctx, const cb_cloud* pts, float* centroids, size_t k, size_t max_iter, float tol,
                      uint64_t* labels, cb_kmeans_result* res) {
  CB_CHECK(ctx && pts && centroids && k > 0, CB_ERR_INVALID, "bad arguments");
  return kmeans_cluster(ctx, KMeansData{pts->d_raw, pts->n, 3}, centroids, k, max_iter, tol, labels, res);
}

int cb_kmeans_assign_vectors(cb_context* ctx, const cb_vectors* vectors, const float* centroids, size_t k,
                             uint64_t* labels, double* sums, uint64_t* counts) {
  CB_TRY(check_vectors(ctx, vectors, centroids, k));
  return kmeans_assign(ctx, KMeansData{vectors->d_raw, vectors->n, vectors->D}, centroids, k, labels, sums, counts);
}

int cb_kmeans_cluster_vectors(cb_context* ctx, const cb_vectors* vectors, float* centroids, size_t k, size_t max_iter,
                              float tol, uint64_t* labels, cb_kmeans_result* res) {
  CB_TRY(check_vectors(ctx, vectors, centroids, k));
  return kmeans_cluster(ctx, KMeansData{vectors->d_raw, vectors->n, vectors->D}, centroids, k, max_iter, tol, labels,
                        res);
}

}  // extern "C"
