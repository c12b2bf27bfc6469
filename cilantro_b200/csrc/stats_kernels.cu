// First and second moments of a point set (product code, sm_90a).
// Replaces the two serial passes of Covariance::operator() (core/covariance.hpp:64-76) and the
// rowwise().mean() of the ICP constructors (icp_single_transform_combined_metric.hpp:51-58) with one
// streaming pass over the packed xyz array: HBM-bound, 12 B/point.
#include "cb_internal.hpp"
#include "reduce.cuh"
#include "stats_kernels.cuh"
#include <algorithm>

namespace cb {

namespace {

// result[0] = n, [1..3] = sum (p - c), [4..9] = sum (p - c)(p - c)^T upper triangle (xx xy xz yy yz zz).
// kFiniteOnly: points with a NaN / Inf coordinate are skipped (n counts the finite ones) - the ICP pivots, which must
// stay finite whatever the cloud holds; otherwise every point counts, as in Covariance::operator().
template <bool kFiniteOnly>
__global__ void __launch_bounds__(kReduceBlock) moments_kernel(const float* __restrict__ raw, size_t n, float cx,
                                                               float cy, float cz, const ReduceScratch rs) {
  double acc[kMomentValues];
#pragma unroll
  for (int i = 0; i < kMomentValues; i++) acc[i] = 0.0;
  auto add = [&](float px, float py, float pz) {
    if (kFiniteOnly && !(isfinite(px) && isfinite(py) && isfinite(pz))) return;
    const double x = (double)px - (double)cx, y = (double)py - (double)cy, z = (double)pz - (double)cz;
    acc[0] += 1.0;
    acc[1] += x;
    acc[2] += y;
    acc[3] += z;
    acc[4] += x * x;
    acc[5] += x * y;
    acc[6] += x * z;
    acc[7] += y * y;
    acc[8] += y * z;
    acc[9] += z * z;
  };
  // 4 points = 48 B = three 16-byte loads per thread and trip (the packed xyz stream is 16 B aligned at
  // multiples of 4 points); two groups per trip keep 6 independent LDG.128 in flight per thread.
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t ngroups = n / 4;
  const float4* __restrict__ raw4 = reinterpret_cast<const float4*>(raw);
  size_t gidx = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  for (; gidx + stride < ngroups; gidx += 2 * stride) {
    const float4 a0 = __ldg(raw4 + 3 * gidx), a1 = __ldg(raw4 + 3 * gidx + 1), a2 = __ldg(raw4 + 3 * gidx + 2);
    const size_t h = gidx + stride;
    const float4 b0 = __ldg(raw4 + 3 * h), b1 = __ldg(raw4 + 3 * h + 1), b2 = __ldg(raw4 + 3 * h + 2);
    add(a0.x, a0.y, a0.z); add(a0.w, a1.x, a1.y); add(a1.z, a1.w, a2.x); add(a2.y, a2.z, a2.w);
    add(b0.x, b0.y, b0.z); add(b0.w, b1.x, b1.y); add(b1.z, b1.w, b2.x); add(b2.y, b2.z, b2.w);
  }
  for (; gidx < ngroups; gidx += stride) {
    const float4 a0 = __ldg(raw4 + 3 * gidx), a1 = __ldg(raw4 + 3 * gidx + 1), a2 = __ldg(raw4 + 3 * gidx + 2);
    add(a0.x, a0.y, a0.z); add(a0.w, a1.x, a1.y); add(a1.z, a1.w, a2.x); add(a2.y, a2.z, a2.w);
  }
  // tail (n % 4 points)
  for (size_t i = ngroups * 4 + blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += stride)
    add(raw[3 * i], raw[3 * i + 1], raw[3 * i + 2]);
  grid_reduce<kMomentValues>(acc, rs);
}

}  // namespace

int launch_moments(cb_context* ctx, const float* d_raw, size_t n, const float* shift3, bool finite_only) {
  // persistent grid: a whole number of resident blocks per SM (occupancy API), 8 points per thread and trip
  static int per_sm[2] = {0, 0};
  int& psm = per_sm[finite_only ? 1 : 0];
  if (psm == 0) {
    int v = 0;
    const cudaError_t e = finite_only ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, moments_kernel<true>, kReduceBlock, 0)
                                      : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, moments_kernel<false>, kReduceBlock, 0);
    if (e != cudaSuccess || v < 1) v = 4;
    psm = v;
  }
  int blocks = (int)std::max<size_t>(
      1, std::min<size_t>((size_t)ctx->sm_count * psm, (n / 8 + kReduceBlock - 1) / kReduceBlock + 1));
  ReduceScratch rs;
  CB_TRY(get_reduce_scratch(ctx, blocks, kMomentValues, &rs));
  if (finite_only)
    moments_kernel<true><<<blocks, kReduceBlock, 0, ctx->stream>>>(d_raw, n, shift3[0], shift3[1], shift3[2], rs);
  else
    moments_kernel<false><<<blocks, kReduceBlock, 0, ctx->stream>>>(d_raw, n, shift3[0], shift3[1], shift3[2], rs);
  ctx->launches += 1;
  CB_CUDA(cudaGetLastError());
  return CB_OK;
}

}  // namespace cb
