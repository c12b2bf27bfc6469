// k-means over D-dimensional rows: fused assignment + centroid-sum kernel (product code, sm_90a).
//
// KMeans<float, D>::cluster_ (clustering/kmeans.hpp:67-194), brute-force branch, for D != 3 (D = 3 runs
// kmeans_assign_kernel of kmeans.cu on the same bytes). The Lloyd loop around it is kmeans.cu's.
// Arithmetic contract (DESIGN §4.17): d = c - p per component in fp32, then the right fold without FMA,
//   acc = d[D-1]^2;  for j = D-2 .. 0:  acc = d[j]^2 + acc
// and the strict-'<' scan over ascending j from +inf (lowest j wins ties, label 0 when no d2 is below +inf).
// Bound: FP32 issue, 3 N K D operations (sub, mul, add). A block takes a tile of 128 points against tiles of
// 128 centroids; each thread keeps an 8 x 8 micro-tile of fold accumulators in registers, fed by four LDS.128
// per dimension from chunks of 16 dimensions staged transposed in shared memory, highest chunk first.
// A row with a non-finite component gets label 0 (no d2 of it is below +inf) and adds to no sum or count.
#include "cb_internal.hpp"
#include "launch.cuh"
#include <algorithm>

using namespace cb;

namespace {

constexpr int kThreads = 256;       // 16 x 16 threads; thread (ty, tx) owns 8 points x 8 centroids of a tile
constexpr int kTile = 128;          // points and centroids per tile
constexpr int kDChunk = 16;         // dimensions per staged chunk
constexpr int kStride = kTile + 4;  // padded row: stays 16-byte aligned, halves the transposed-store conflicts

struct Staging {
  float p[kDChunk][kStride];  // points of the tile, [dimension][point]
  float c[kDChunk][kStride];  // centroids of the tile, [dimension][centroid]
  uint32_t label[kTile];
  int bad[kTile];  // the point has a non-finite component
};

// rows [r0, r0 + rows) x dimensions [d0, d0 + dn) of a row-major n x D array into s[dd][r]; rows past `rows` read 0
__device__ __forceinline__ void stage(float (*s)[kStride], const float* __restrict__ src, size_t r0, int rows, int D,
                                      int d0, int dn, int* bad) {
  for (int e = threadIdx.x; e < kTile * dn; e += kThreads) {
    const int r = e / dn, dd = e - r * dn;
    float v = 0.f;
    if (r < rows) {
      v = src[(r0 + r) * (size_t)D + d0 + dd];
      if (bad && !isfinite(v)) bad[r] = 1;
    }
    s[dd][r] = v;
  }
}

// the micro-tile's u-th point / v-th centroid within its tile (ascending in u and v)
__device__ __forceinline__ int slot(int t, int u) { return u < 4 ? t * 4 + u : 64 + t * 4 + (u - 4); }

// sums layout: K x (D + 1) doubles (D coordinate sums, then the count)
template <bool kSmemSums>
__global__ void __launch_bounds__(kThreads, 2)
    kmeans_features_assign_kernel(const float* __restrict__ raw, size_t n, int D, const float* __restrict__ cent, int K,
                                  uint32_t* __restrict__ labels, double* __restrict__ sums,
                                  unsigned int* __restrict__ changed) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Staging& st = *reinterpret_cast<Staging*>(smem_raw);
  double* s_sums = reinterpret_cast<double*>(smem_raw + sizeof(Staging));  // K x (D + 1) if kSmemSums
  const int W = D + 1;
  if (kSmemSums) {
    for (int j = threadIdx.x; j < K * W; j += kThreads) s_sums[j] = 0.0;
  }
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  unsigned int any_changed = 0;
  const size_t ntiles = (n + kTile - 1) / kTile;
  for (size_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const size_t base = t * kTile;
    const int rows = (int)min((size_t)kTile, n - base);
    if (threadIdx.x < kTile) st.bad[threadIdx.x] = 0;
    float best[8];
    int bi[8];
#pragma unroll
    for (int u = 0; u < 8; u++) {
      best[u] = __int_as_float(0x7f800000);  // +inf
      bi[u] = 0x7fffffff;                     // none below +inf yet
    }
    for (int c0 = 0; c0 < K; c0 += kTile) {
      const int cn = min(kTile, K - c0);
      float acc[8][8];
#pragma unroll
      for (int u = 0; u < 8; u++)
#pragma unroll
        for (int v = 0; v < 8; v++) acc[u][v] = 0.f;  // 0 + d[D-1]^2 is d[D-1]^2 exactly
      for (int hi = D; hi > 0; hi -= kDChunk) {
        const int lo = max(0, hi - kDChunk), dn = hi - lo;
        __syncthreads();
        stage(st.p, raw, base, rows, D, lo, dn, c0 == 0 ? st.bad : nullptr);
        stage(st.c, cent, (size_t)c0, cn, D, lo, dn, nullptr);
        __syncthreads();
#pragma unroll 2
        for (int dd = dn - 1; dd >= 0; dd--) {
          const float4 pa = *reinterpret_cast<const float4*>(&st.p[dd][ty * 4]);
          const float4 pb = *reinterpret_cast<const float4*>(&st.p[dd][64 + ty * 4]);
          const float4 ca = *reinterpret_cast<const float4*>(&st.c[dd][tx * 4]);
          const float4 cb = *reinterpret_cast<const float4*>(&st.c[dd][64 + tx * 4]);
          const float p[8] = {pa.x, pa.y, pa.z, pa.w, pb.x, pb.y, pb.z, pb.w};
          const float c[8] = {ca.x, ca.y, ca.z, ca.w, cb.x, cb.y, cb.z, cb.w};
#pragma unroll
          for (int u = 0; u < 8; u++)
#pragma unroll
            for (int v = 0; v < 8; v++) {
              const float d = __fsub_rn(c[v], p[u]);
              acc[u][v] = __fadd_rn(__fmul_rn(d, d), acc[u][v]);
            }
        }
      }
      // this thread's centroids of the tile, ascending j, strict '<' (kmeans.hpp:108-113)
#pragma unroll
      for (int v = 0; v < 8; v++) {
        const int j = slot(tx, v);
        if (j >= cn) continue;
#pragma unroll
        for (int u = 0; u < 8; u++)
          if (acc[u][v] < best[u]) {
            best[u] = acc[u][v];
            bi[u] = c0 + j;
          }
      }
    }
    // the 16 threads of a point row hold disjoint centroid sets: smallest d2, then lowest j
#pragma unroll
    for (int u = 0; u < 8; u++) {
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best[u], o);
        const int oj = __shfl_xor_sync(0xffffffffu, bi[u], o);
        if (ob < best[u] || (ob == best[u] && oj < bi[u])) {
          best[u] = ob;
          bi[u] = oj;
        }
      }
      if (tx == 0) st.label[slot(ty, u)] = bi[u] == 0x7fffffff ? 0u : (uint32_t)bi[u];
    }
    __syncthreads();
    double* S = kSmemSums ? s_sums : sums;
    if (threadIdx.x < rows) {
      const size_t i = base + threadIdx.x;
      const uint32_t lab = st.label[threadIdx.x];
      if (labels[i] != lab) any_changed = 1;
      labels[i] = lab;
      if (!st.bad[threadIdx.x]) atomicAdd(S + (size_t)lab * W + D, 1.0);
    }
    for (int e = threadIdx.x; e < rows * D; e += kThreads) {
      const int r = e / D, j = e - r * D;
      if (!st.bad[r]) atomicAdd(S + (size_t)st.label[r] * W + j, (double)raw[(base + r) * (size_t)D + j]);
    }
    __syncthreads();
  }
  if (kSmemSums) {
    __syncthreads();
    for (int j = threadIdx.x; j < K * W; j += kThreads) {
      const double v = s_sums[j];
      if (v != 0.0) atomicAdd(sums + j, v);
    }
  }
  if (__syncthreads_or(any_changed) && threadIdx.x == 0) atomicOr(changed, 1u);
}

}  // namespace

namespace cb {

int kmeans_features_assign(cb_context* ctx, const float* raw, size_t n, int D, const float* cent, size_t K,
                           uint32_t* labels, double* sums, unsigned int* changed) {
  const size_t sums_bytes = K * (size_t)(D + 1) * sizeof(double);
  const bool use_smem = sums_bytes <= kKMeansSmemSumsBytes;
  const size_t smem = sizeof(Staging) + (use_smem ? sums_bytes : 0);
  auto kern = use_smem ? kmeans_features_assign_kernel<true> : kmeans_features_assign_kernel<false>;
  CB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  CB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, smem));
  per_sm = std::max(1, per_sm);
  return launch(ctx, kern, grid_for(ctx, n, kTile, per_sm), kThreads, smem, raw, n, D, cent, (int)K, labels, sums,
                changed);
}

}  // namespace cb
