// General-k nearest neighbours over the grid (product code, sm_90a).
// Replaces the batched KDTree::kNNInRadiusSearch / kNNSearch (core/kd_tree.hpp:215-318) for k <= 256 (the k-best list is a
// per-thread array: registers for small k, L1-resident local memory for large k; the reference is unbounded in k):
// same shell sweep as nn_search.cuh, with a per-thread sorted list of the k best (d2, index) pairs
// whose worst entry plays the role of nanoflann's worstDist() (kd_tree.hpp:101).
#include "cb_internal.hpp"
#include "grid_sweep.cuh"
#include "kbest.cuh"
#include "launch.cuh"
#include "radius_lists.cuh"
#include <algorithm>
#include <vector>

using namespace cb;

namespace {

constexpr int kMaxK = kKBestMaxK;
constexpr int kBlock = 128;

template <int K>
__global__ void __launch_bounds__(kBlock) knn_k_kernel(const GridView g, const float4* __restrict__ qry, uint32_t nq,
                                                       const Rigid T, int k, float max_d2, int* __restrict__ out_idx,
                                                       float* __restrict__ out_d2, uint32_t* __restrict__ out_cnt) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t qi = blockIdx.x * blockDim.x + threadIdx.x; qi < nq; qi += stride) {
    const float4 s = __ldg(qry + qi);
    const int oi = __float_as_int(s.w);
    float qx, qy, qz;
    rule::transform_point(T, s.x, s.y, s.z, qx, qy, qz);
    float bd[K];
    int bi[K];
    int count = 0;
    // bound = current worst admissible squared distance (strict): max_d2 until k found
    auto bound = [&]() { return (count == k) ? bd[k - 1] : max_d2; };
    auto scan = [&](uint32_t b, uint32_t e) {
      for (uint32_t j = b; j < e; ++j) {
        const float4 p = __ldg(g.pts + j);
        const float r = rule::contract_d2(qx, qy, qz, p.x, p.y, p.z);
        if (r < max_d2) kbest_insert<K>(bd, bi, k, count, r, __float_as_int(p.w));
      }
    };
    grid_sweep(g, qx, qy, qz, bound, scan, [&]() { count = 0; }, (uint32_t)k);
    for (int j = 0; j < k; j++) {
      out_idx[(size_t)oi * k + j] = (j < count) ? bi[j] : -1;
      out_d2[(size_t)oi * k + j] = (j < count) ? bd[j] : max_d2;
    }
    if (out_cnt) out_cnt[oi] = (uint32_t)count;
  }
}

}  // namespace

extern "C" int cb_knn_radius(cb_context* ctx, const cb_cloud* ref, const cb_cloud* qry, const float* T12, int k,
                             float max_d2, int64_t* idx, float* d2, uint32_t* counts) {
  CB_CHECK(ctx && ref && qry && idx && d2, CB_ERR_INVALID, "null argument");
  CB_CHECK(k >= 1 && k <= kMaxK, CB_ERR_UNSUPPORTED, "k must be in [1, 256]");
  CB_CHECK(ref->ctx == ctx && qry->ctx == ctx, CB_ERR_INVALID, "cloud belongs to another context");
  CB_CUDA(cudaSetDevice(ctx->device));
  CB_TRY(ensure_index(const_cast<cb_cloud*>(ref)));
  CB_TRY(ensure_index(const_cast<cb_cloud*>(qry)));
  const size_t nq = qry->n;
  if (nq == 0) return CB_OK;
  const Rigid T = rigid_from_t12(T12);
  DeviceScope scope(ctx);
  int* d_idx = nullptr;
  float* d_d2 = nullptr;
  uint32_t* d_cnt = nullptr;
  CB_TRY(scope.alloc(&d_idx, nq * k));
  CB_TRY(scope.alloc(&d_d2, nq * k));
  CB_TRY(scope.alloc(&d_cnt, nq));
  auto kernel = knn_k_kernel<256>;
  if (k <= 4)
    kernel = knn_k_kernel<4>;
  else if (k <= 16)
    kernel = knn_k_kernel<16>;
  else if (k <= 32)
    kernel = knn_k_kernel<32>;
  else if (k <= 64)
    kernel = knn_k_kernel<64>;
  else if (k <= 128)
    kernel = knn_k_kernel<128>;
  CB_TRY(launch(ctx, kernel, grid_for(ctx, nq, kBlock), kBlock, 0, grid_view(ref), qry->d_pts, (uint32_t)nq, T, k,
                max_d2, d_idx, d_d2, d_cnt));
  std::vector<int> h_idx(nq * k);
  CB_CUDA(cudaMemcpyAsync(h_idx.data(), d_idx, nq * k * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaMemcpyAsync(d2, d_d2, nq * k * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  if (counts) CB_CUDA(cudaMemcpyAsync(counts, d_cnt, nq * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  for (size_t i = 0; i < nq * k; i++) idx[i] = h_idx[i] < 0 ? -1 : (int64_t)h_idx[i] + (int64_t)ref->index_offset;
  return CB_OK;
}

// ---- radius neighbourhoods (variable length): radius_kernel + segment_heapsort_kernel (radius_lists.cuh) ----------

extern "C" int cb_radius_search(cb_context* ctx, const cb_cloud* ref, const cb_cloud* qry, const float* T12,
                                float radius2, uint64_t* offsets, int64_t* idx, float* d2, size_t capacity,
                                size_t* total) {
  CB_CHECK(ctx && ref && qry && offsets && total, CB_ERR_INVALID, "null argument");
  CB_CHECK(ref->ctx == ctx && qry->ctx == ctx, CB_ERR_INVALID, "cloud belongs to another context");
  CB_CUDA(cudaSetDevice(ctx->device));
  CB_TRY(ensure_index(const_cast<cb_cloud*>(ref)));
  CB_TRY(ensure_index(const_cast<cb_cloud*>(qry)));
  const size_t nq = qry->n;
  *total = 0;
  offsets[0] = 0;
  if (nq == 0) return CB_OK;
  const Rigid T = rigid_from_t12(T12);
  DeviceScope scope(ctx);
  uint32_t* d_off = nullptr;
  CB_TRY(scope.alloc(&d_off, nq + 2));
  CB_CUDA(cudaMemsetAsync(d_off, 0, (nq + 2) * sizeof(uint32_t), ctx->stream));
  const int blocks = grid_for(ctx, nq, kBlock);
  const GridView g = grid_view(ref);
  CB_TRY(launch(ctx, radius_kernel<false>, blocks, kBlock, 0, g, qry->d_pts, (uint32_t)nq, T, radius2, d_off, nullptr,
                nullptr, nullptr));
  // counts are 32-bit: sum them on the host in 64 bits before trusting the 32-bit scan
  std::vector<uint32_t> h_cnt(nq);
  CB_CUDA(cudaMemcpyAsync(h_cnt.data(), d_off, nq * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  uint64_t sum = 0;
  for (size_t i = 0; i < nq; i++) {
    offsets[i] = sum;
    sum += h_cnt[i];
  }
  offsets[nq] = sum;
  *total = (size_t)sum;
  if (sum == 0 || !idx || !d2 || capacity < sum)
    return CB_OK;  // sizing call, or the caller's buffers are too small: *total says what is needed
  CB_CHECK(sum < (1ull << 32), CB_ERR_UNSUPPORTED, "radius search: more than 2^32 - 1 neighbour pairs in one call");
  CB_TRY(exclusive_scan_u32(ctx, d_off, nq + 1, 0u));
  int* d_idx = nullptr;
  float* d_d2 = nullptr;
  CB_TRY(scope.alloc(&d_idx, sum));
  CB_TRY(scope.alloc(&d_d2, sum));
  CB_TRY(launch(ctx, radius_kernel<true>, blocks, kBlock, 0, g, qry->d_pts, (uint32_t)nq, T, radius2, nullptr, d_off,
                d_idx, d_d2));
  CB_TRY(launch(ctx, segment_heapsort_kernel, blocks, kBlock, 0, d_off, (uint32_t)nq, d_idx, d_d2));
  std::vector<int> h_idx(sum);
  CB_CUDA(cudaMemcpyAsync(h_idx.data(), d_idx, sum * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaMemcpyAsync(d2, d_d2, sum * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  for (size_t i = 0; i < sum; i++) idx[i] = (int64_t)h_idx[i] + (int64_t)ref->index_offset;
  return CB_OK;
}
