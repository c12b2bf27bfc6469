// Stable LSD radix sort of (uint64 key, uint32 value) pairs, 8 bits per pass (product code, sm_90a).
// Used by the voxel-grid downsampler (bin key -> point index) where the number of bins is unbounded and a
// dense counter table (grid_index.cu) is not an option. HBM-bound integer work: per pass one histogram
// read (8 B/elem) and one scatter pass (12 B read + 12 B written per element); only the passes the key
// range needs are run.
//
// Per pass: radix_hist_kernel counts the digit of every element of a 4096-element tile into a
// digit-major table hist[digit][tile]; one exclusive scan of that table (grid_index.cu) turns it into the
// global destination of the first element of every (digit, tile); radix_scatter_kernel re-reads the tile,
// splits it into 8 contiguous warp slices, ranks equal digits inside a warp round with __match_any_sync
// and keeps a running destination per (warp, digit) in shared memory — the element order inside equal
// digits is the input order (stable), which the downsampler relies on: points of one bin stay sorted by
// their original index.
#include "cb_internal.hpp"
#include "launch.cuh"
#include <algorithm>

namespace cb {

namespace {

constexpr int kSortThreads = 256;
constexpr int kSortWarps = kSortThreads / 32;
constexpr int kRounds = 16;                                // 32-element rounds per warp
constexpr int kWarpItems = 32 * kRounds;                   // 512
constexpr int kTile = kSortWarps * kWarpItems;             // 4096 elements per block
constexpr int kDigits = 256;

__global__ void __launch_bounds__(kSortThreads) radix_hist_kernel(const uint64_t* __restrict__ keys, size_t n, int shift,
                                                                  uint32_t* __restrict__ hist, uint32_t ntiles) {
  __shared__ uint32_t cnt[kDigits];
  cnt[threadIdx.x] = 0;
  __syncthreads();
  const size_t base = (size_t)blockIdx.x * kTile;
#pragma unroll 4
  for (int k = threadIdx.x; k < kTile; k += kSortThreads) {
    const size_t i = base + k;
    if (i < n) atomicAdd(&cnt[(uint32_t)(keys[i] >> shift) & 0xffu], 1u);
  }
  __syncthreads();
  hist[(size_t)threadIdx.x * ntiles + blockIdx.x] = cnt[threadIdx.x];
}

__global__ void __launch_bounds__(kSortThreads) radix_scatter_kernel(const uint64_t* __restrict__ keys,
                                                                     const uint32_t* __restrict__ vals, size_t n,
                                                                     int shift, const uint32_t* __restrict__ offs,
                                                                     uint32_t ntiles, uint64_t* __restrict__ out_keys,
                                                                     uint32_t* __restrict__ out_vals) {
  __shared__ uint32_t dest[kSortWarps][kDigits];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int w = 0; w < kSortWarps; w++) dest[w][threadIdx.x] = 0;
  __syncthreads();
  const size_t wbase = (size_t)blockIdx.x * kTile + (size_t)warp * kWarpItems;
  // A: digit counts of this warp's slice
  for (int r = 0; r < kRounds; r++) {
    const size_t i = wbase + (size_t)r * 32 + lane;
    if (i < n) atomicAdd(&dest[warp][(uint32_t)(keys[i] >> shift) & 0xffu], 1u);
  }
  __syncthreads();
  // B: counts -> running global destinations (thread d owns digit d)
  {
    uint32_t run = offs[(size_t)threadIdx.x * ntiles + blockIdx.x];
    for (int w = 0; w < kSortWarps; w++) {
      const uint32_t c = dest[w][threadIdx.x];
      dest[w][threadIdx.x] = run;
      run += c;
    }
  }
  __syncthreads();
  // C: ranked scatter, round by round in input order
  for (int r = 0; r < kRounds; r++) {
    const size_t i = wbase + (size_t)r * 32 + lane;
    const bool live = i < n;
    const unsigned active = __ballot_sync(0xffffffffu, live);
    if (live) {
      const uint64_t key = keys[i];
      const uint32_t val = vals[i];
      const uint32_t d = (uint32_t)(key >> shift) & 0xffu;
      const unsigned peers = __match_any_sync(active, d);
      const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
      const uint32_t pos = dest[warp][d] + rank;
      __syncwarp(active);
      if (rank == 0) dest[warp][d] += __popc(peers);
      __syncwarp(active);
      out_keys[pos] = key;
      out_vals[pos] = val;
    }
  }
}

}  // namespace

int radix_sort_pairs_u64(cb_context* ctx, uint64_t* d_keys, uint32_t* d_vals, uint64_t* d_keys_tmp,
                         uint32_t* d_vals_tmp, size_t n, int bits) {
  if (n <= 1 || bits <= 0) return CB_OK;
  CB_CHECK(n < (1ull << 32), CB_ERR_INVALID, "radix sort: more than 2^32 - 1 elements");
  const uint32_t ntiles = (uint32_t)((n + kTile - 1) / kTile);
  const size_t hn = (size_t)kDigits * ntiles;
  DeviceScope scope(ctx);
  uint32_t* d_hist = nullptr;
  CB_TRY(scope.alloc(&d_hist, hn + 1));
  uint64_t* kin = d_keys;
  uint32_t* vin = d_vals;
  uint64_t* kout = d_keys_tmp;
  uint32_t* vout = d_vals_tmp;
  const int passes = (std::min(bits, 64) + 7) / 8;
  for (int p = 0; p < passes; p++) {
    const int shift = 8 * p;
    CB_TRY(launch(ctx, radix_hist_kernel, ntiles, kSortThreads, 0, kin, n, shift, d_hist, ntiles));
    CB_TRY(exclusive_scan_u32(ctx, d_hist, hn, (uint32_t)n));
    CB_TRY(launch(ctx, radix_scatter_kernel, ntiles, kSortThreads, 0, kin, vin, n, shift, d_hist, ntiles, kout, vout));
    std::swap(kin, kout);
    std::swap(vin, vout);
  }
  if (kin != d_keys) {
    CB_CUDA(cudaMemcpyAsync(d_keys, kin, n * sizeof(uint64_t), cudaMemcpyDeviceToDevice, ctx->stream));
    CB_CUDA(cudaMemcpyAsync(d_vals, vin, n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->stream));
  }
  return CB_OK;
}

}  // namespace cb
