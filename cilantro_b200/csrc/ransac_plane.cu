// Plane RANSAC on the device (product code, sm_90a). DESIGN §4.12.
//
// Replaces RandomSampleConsensusBase::estimate (model_estimation/ransac_base.hpp:64-131) with
// HyperplaneRANSACEstimator<float, 3> (ransac_hyperplane_estimator.hpp). The reference fits each sample with a PCA,
// then streams the whole cloud once per hypothesis in computeResiduals (:47-55) and scans the residual vector
// serially. Here the samples are drawn on the host in the reference's order, fitted on the device
// (plane_fit_kernel, the closed form of plane_fit.hpp), and a batch of hypotheses is scored in one pass over the
// cloud (plane_score_kernel): each thread keeps kPts points in registers, the planes of the batch sit in shared
// memory, and only the batch's inlier counts leave the chip. Bound: instruction issue, 9.6 SASS instructions per
// point-hypothesis (3 FMUL, 3 FADD, FSETP + SEL for the mask, the count's share of an IADD3, and the per-plane
// shared-memory and warp-reduction work spread over the 8 points).
//
// Residual contract: r = |((n0 x) + ((n1 y) + (n2 z))) + d| with every operation rounded on its own; inlier iff
// r <= thresh. Points past the end of the cloud are loaded as NaN, which is never an inlier, so the inner loop
// carries no bounds test.
#include "cb_internal.hpp"
#include "host_solve.hpp"
#include "launch.cuh"
#include "plane_fit.hpp"
#include "ransac_loop.hpp"
#include "reduce.cuh"
#include "stats_kernels.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <vector>

using namespace cb;

namespace {

constexpr int kBlock = 256;
constexpr int kWarps = kBlock / 32;
constexpr int kPts = 8;            // points per thread in registers
constexpr int kWarpTile = 32 * kPts;
constexpr int kMaxBatch = 1024;   // planes per launch: all of them staged in shared memory (16 KB + 32 KB counters)
constexpr int kFirstBatch = 64;   // hypotheses of the loop's first batch; doubled per batch up to kMaxBatch

__device__ __forceinline__ float plane_residual(const float4 P, float x, float y, float z) {
  return fabsf(__fadd_rn(__fadd_rn(__fmul_rn(P.x, x), __fadd_rn(__fmul_rn(P.y, y), __fmul_rn(P.z, z))), P.w));
}

// 0xffffffff (-1) iff r <= thresh: one FSET, so that counting an inlier costs one more IADD (a C comparison
// compiles to FSETP + IADD + a predicated move)
__device__ __forceinline__ int inlier_mask(float r, float thresh) {
  int m;
  asm("set.le.s32.f32 %0, %1, %2;" : "=r"(m) : "f"(r), "f"(thresh));
  return m;
}

// counts[h] += inliers of plane h; counts zeroed by the caller. A warp owns tiles of 32 x kPts consecutive points
// (tile t, t + total warps, ...), so the work of an SM differs from the mean by at most one tile per warp.
__global__ void __launch_bounds__(kBlock) plane_score_kernel(const float* __restrict__ raw, size_t n,
                                                             const float4* __restrict__ planes, int H, float thresh,
                                                             uint32_t* __restrict__ counts) {
  __shared__ float4 s_pl[kMaxBatch];
  __shared__ uint32_t s_cnt[kWarps][kMaxBatch];  // one row per warp: plain adds, no shared atomics
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int h = threadIdx.x; h < H; h += kBlock) {
    s_pl[h] = planes[h];
    for (int w = 0; w < kWarps; w++) s_cnt[w][h] = 0;
  }
  __syncthreads();
  const size_t ntiles = (n + kWarpTile - 1) / kWarpTile;
  const size_t warps = (size_t)gridDim.x * kWarps;
  const float nan = __int_as_float(0x7fc00000);
  uint32_t* row = s_cnt[warp];
  for (size_t t = (size_t)blockIdx.x * kWarps + warp; t < ntiles; t += warps) {
    float x[kPts], y[kPts], z[kPts];
#pragma unroll
    for (int u = 0; u < kPts; u++) {
      const size_t i = t * kWarpTile + (size_t)u * 32 + lane;
      const bool ok = i < n;
      x[u] = ok ? raw[3 * i] : nan;
      y[u] = ok ? raw[3 * i + 1] : nan;
      z[u] = ok ? raw[3 * i + 2] : nan;
    }
    for (int h = 0; h < H; h++) {
      const float4 P = s_pl[h];
      int c = 0;
#pragma unroll
      for (int u = 0; u < kPts; u++) c -= inlier_mask(plane_residual(P, x[u], y[u], z[u]), thresh);
      c = __reduce_add_sync(0xffffffffu, c);
      if (lane == 0) row[h] += (uint32_t)c;
    }
  }
  __syncthreads();
  for (int h = threadIdx.x; h < H; h += kBlock) {
    uint32_t c = 0;
    for (int w = 0; w < kWarps; w++) c += s_cnt[w][h];
    if (c) atomicAdd(counts + h, c);
  }
}

// estimateModel(sample) (ransac_hyperplane_estimator.hpp:36-42) for H samples of sample_size (<= 3) indices each,
// stored with a stride of 3
__global__ void plane_fit_kernel(const float* __restrict__ raw, const uint32_t* __restrict__ idx, int H,
                                 int sample_size, float4* __restrict__ planes) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= H) return;
  float p[9];
  for (int i = 0; i < sample_size; i++) {
    const size_t j = idx[3 * (size_t)h + i];
    for (int r = 0; r < 3; r++) p[3 * i + r] = raw[3 * j + r];
  }
  float out[4];
  plane::fit(p, sample_size, out);
  planes[h] = make_float4(out[0], out[1], out[2], out[3]);
}

// residuals (may be null) and the inlier flags of one plane; flags[n] = 0 (the scan turns it into the count)
__global__ void plane_residual_kernel(const float* __restrict__ raw, size_t n, const float4 P, float thresh,
                                      float* __restrict__ res, uint32_t* __restrict__ flags) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i <= n; i += (size_t)gridDim.x * blockDim.x) {
    if (i == n) {
      flags[n] = 0u;
      continue;
    }
    const float r = plane_residual(P, raw[3 * i], raw[3 * i + 1], raw[3 * i + 2]);
    if (res) res[i] = r;
    flags[i] = r <= thresh ? 1u : 0u;
  }
}

// The moments of moments_kernel (count, sum (p - c), upper triangle of sum (p - c)(p - c)^T) over the points with
// |n.p + d| <= thresh, the predicate that counted the hypothesis's inliers
__global__ void __launch_bounds__(kReduceBlock) plane_moments_kernel(const float* __restrict__ raw, size_t n,
                                                                     const float4 P, float thresh, float cx, float cy,
                                                                     float cz, const ReduceScratch rs) {
  double acc[kMomentValues];
#pragma unroll
  for (int i = 0; i < kMomentValues; i++) acc[i] = 0.0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float px = raw[3 * i], py = raw[3 * i + 1], pz = raw[3 * i + 2];
    if (!(plane_residual(P, px, py, pz) <= thresh)) continue;
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
  }
  grid_reduce<kMomentValues>(acc, rs);
}

int check_cloud(cb_context* ctx, const cb_cloud* cloud) {
  CB_CHECK(ctx && cloud, CB_ERR_INVALID, "null argument");
  CB_CHECK(cloud->ctx == ctx, CB_ERR_INVALID, "cloud belongs to another context");
  CB_CHECK(cloud->index_offset == 0, CB_ERR_UNSUPPORTED, "plane RANSAC runs on a whole cloud (index_offset must be 0)");
  CB_CHECK(cloud->n < 0xffffffffull, CB_ERR_UNSUPPORTED, "plane RANSAC supports fewer than 2^32 - 1 points");
  CB_CUDA(cudaSetDevice(ctx->device));
  return CB_OK;
}

// counts (device, H <= kMaxBatch) of the planes already in device memory; zeroed here
int score_planes(cb_context* ctx, const cb_cloud* cloud, const float4* d_planes, int H, float thresh,
                 uint32_t* d_counts) {
  CB_CUDA(cudaMemsetAsync(d_counts, 0, (size_t)H * sizeof(uint32_t), ctx->stream));
  if (cloud->n == 0 || H == 0) return CB_OK;
  static int per_sm = 0;
  if (per_sm == 0) {
    int v = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, plane_score_kernel, kBlock, 0) != cudaSuccess || v < 1) v = 1;
    per_sm = v;
  }
  const size_t ntiles = (cloud->n + kWarpTile - 1) / kWarpTile;
  return launch(ctx, plane_score_kernel, grid_for(ctx, ntiles, kWarps, per_sm), kBlock, 0, cloud->d_raw, cloud->n,
                d_planes, H, thresh, d_counts);
}

int fit_planes(cb_context* ctx, const cb_cloud* cloud, const uint32_t* d_idx, int H, int sample_size, float4* d_planes) {
  if (H == 0) return CB_OK;
  return launch(ctx, plane_fit_kernel, (H + 127) / 128, 128, 0, cloud->d_raw, d_idx, H, sample_size, d_planes);
}

// moments of the points within thresh of the plane about the pivot c (synchronises the stream)
int plane_moments(cb_context* ctx, const cb_cloud* cloud, const float* plane4, float thresh, const float* c,
                  double* m) {
  const size_t n = cloud->n;
  const int blocks = grid_for(ctx, n, kReduceBlock, 4);
  ReduceScratch rs;
  CB_TRY(get_reduce_scratch(ctx, blocks, kMomentValues, &rs));
  const float4 P = make_float4(plane4[0], plane4[1], plane4[2], plane4[3]);
  CB_TRY(launch(ctx, plane_moments_kernel, blocks, kReduceBlock, 0, cloud->d_raw, n, P, thresh, c[0], c[1], c[2], rs));
  return fetch_result(ctx, kMomentValues, false, m);
}

// Re-estimation (ransac_base.hpp:118-120): the PCA of the inliers of plane4 (expected_count of them), the normal =
// the third eigenvector, offset = -(n . mean) in fp32 (ransac_hyperplane_estimator.hpp:103-110). The moments are
// summed in double about a pivot (a first pass about the origin gives it), like cb_pca.
int reestimate(cb_context* ctx, const cb_cloud* cloud, const float* plane4, float thresh, size_t expected_count,
               float* out) {
  double m[kMomentValues];
  const float zero[3] = {0.f, 0.f, 0.f};
  CB_TRY(plane_moments(ctx, cloud, plane4, thresh, zero, m));
  CB_CHECK(m[0] == (double)expected_count, CB_ERR_CUDA, "internal: re-estimation selected a different inlier set");
  const float nan = std::numeric_limits<float>::quiet_NaN();
  if (m[0] < 2.0) {  // covariance.hpp:35-38
    for (int r = 0; r < 4; r++) out[r] = nan;
    return CB_OK;
  }
  float pivot[3];
  for (int r = 0; r < 3; r++) pivot[r] = (float)(m[1 + r] / m[0]);
  CB_TRY(plane_moments(ctx, cloud, plane4, thresh, pivot, m));
  const double cnt = m[0];
  const double s1[3] = {m[1], m[2], m[3]};
  const double s2[3][3] = {{m[4], m[5], m[6]}, {m[5], m[7], m[8]}, {m[6], m[8], m[9]}};
  float mean[3];
  double cov[9];
  for (int r = 0; r < 3; r++) mean[r] = (float)((double)pivot[r] + s1[r] / cnt);
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) cov[r * 3 + c] = (double)(float)((s2[r][c] - s1[r] * s1[c] / cnt) / (cnt - 1.0));
  float evals[3], evecs[9];
  pca_from_cov(cov, evals, evecs);  // the eigen-solver sees the fp32 covariance
  const float n0 = evecs[2], n1 = evecs[5], n2 = evecs[8];
  out[0] = n0;
  out[1] = n1;
  out[2] = n2;
  volatile float t1 = n1 * mean[1], t2 = n2 * mean[2], t0 = n0 * mean[0];
  volatile float s12 = t1 + t2;
  volatile float s = t0 + s12;
  out[3] = -s;
  return CB_OK;
}

struct Events {
  cudaEvent_t e[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  int create() {
    for (auto& x : e) CB_CUDA(cudaEventCreate(&x));
    return CB_OK;
  }
  float ms(int a, int b) const {
    float v = 0.f;
    cudaEventElapsedTime(&v, e[a], e[b]);
    return v;
  }
  ~Events() {
    for (auto& x : e)
      if (x) cudaEventDestroy(x);
  }
};

// The plane model of ransac_loop: the samples are fitted (plane_fit_kernel) and scored on the device, and the planes
// come back with the counts. ev.e[0..2] bracket each batch's fit and scoring.
struct PlaneHypotheses {
  cb_context* ctx;
  const cb_cloud* cloud;
  float thresh;
  uint32_t* d_idx;
  float4* d_planes;
  uint32_t* d_counts;
  Events ev;
  std::vector<float> h_planes = std::vector<float>(4 * (size_t)kMaxBatch);
  float best[4];
  double ms_fit = 0.0, ms_score = 0.0;

  int fit(const uint32_t* idx, size_t nb, size_t sample_size) {
    CB_CUDA(cudaEventRecord(ev.e[0], ctx->stream));
    CB_CUDA(cudaMemcpyAsync(d_idx, idx, 3 * nb * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
    CB_TRY(fit_planes(ctx, cloud, d_idx, (int)nb, (int)sample_size, d_planes));
    CB_CUDA(cudaEventRecord(ev.e[1], ctx->stream));
    return CB_OK;
  }
  int score(size_t nb, uint32_t* counts) {
    CB_TRY(score_planes(ctx, cloud, d_planes, (int)nb, thresh, d_counts));
    CB_CUDA(cudaEventRecord(ev.e[2], ctx->stream));
    CB_CUDA(cudaMemcpyAsync(counts, d_counts, nb * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaMemcpyAsync(h_planes.data(), d_planes, nb * sizeof(float4), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    ms_fit += ev.ms(0, 1);
    ms_score += ev.ms(1, 2);
    return CB_OK;
  }
  void keep(size_t b) { std::memcpy(best, &h_planes[4 * b], sizeof(best)); }
};

}  // namespace

extern "C" {

int cb_plane_score(cb_context* ctx, const cb_cloud* cloud, const float* planes4, size_t H, float thresh,
                   uint32_t* counts) {
  CB_TRY(check_cloud(ctx, cloud));
  CB_CHECK(H == 0 || (planes4 && counts), CB_ERR_INVALID, "null argument");
  if (H == 0) return CB_OK;
  DeviceScope scope(ctx);
  float4* d_planes = nullptr;
  uint32_t* d_counts = nullptr;
  const size_t cap = std::min<size_t>(H, kMaxBatch);
  CB_TRY(scope.alloc(&d_planes, cap));
  CB_TRY(scope.alloc(&d_counts, cap));
  for (size_t h0 = 0; h0 < H; h0 += kMaxBatch) {
    const int hn = (int)std::min<size_t>(kMaxBatch, H - h0);
    CB_CUDA(cudaMemcpyAsync(d_planes, planes4 + 4 * h0, (size_t)hn * sizeof(float4), cudaMemcpyHostToDevice, ctx->stream));
    CB_TRY(score_planes(ctx, cloud, d_planes, hn, thresh, d_counts));
    CB_CUDA(cudaMemcpyAsync(counts + h0, d_counts, (size_t)hn * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  return CB_OK;
}

int cb_plane_residuals(cb_context* ctx, const cb_cloud* cloud, const float* plane4, float thresh, float* residuals,
                       uint64_t* inliers, size_t* num_inliers) {
  CB_TRY(check_cloud(ctx, cloud));
  CB_CHECK(plane4, CB_ERR_INVALID, "null argument");
  const size_t n = cloud->n;
  DeviceScope scope(ctx);
  uint32_t* d_flags = nullptr;
  float* d_res = nullptr;
  CB_TRY(scope.alloc(&d_flags, n + 2));
  if (residuals) CB_TRY(scope.alloc(&d_res, n));
  const float4 P = make_float4(plane4[0], plane4[1], plane4[2], plane4[3]);
  if (n)  // n + 1 items: the kernel also writes flags[n]
    CB_TRY(launch(ctx, plane_residual_kernel, grid_for(ctx, n + 1, 256), 256, 0, cloud->d_raw, n, P, thresh, d_res,
                  d_flags));
  return ransac_inliers(ctx, d_flags, d_res, n, 0, residuals, inliers, num_inliers);
}

int cb_ransac_plane(cb_context* ctx, const cb_cloud* cloud, uint32_t seed, size_t inlier_count_thresh,
                    size_t max_iter, float thresh, int re_estimate, cb_ransac_plane_result* res, uint64_t* inliers,
                    float* residuals) {
  CB_TRY(check_cloud(ctx, cloud));
  CB_CHECK(res, CB_ERR_INVALID, "null argument");
  CB_CHECK(ctx->world == 1, CB_ERR_UNSUPPORTED, "cb_ransac_plane runs per process; shard hypotheses with cb_plane_score");
  const uint64_t launches0 = ctx->launches;
  RansacSampler sampler(cloud->n, seed);
  PlaneHypotheses h{ctx, cloud, thresh};
  std::fill(h.best, h.best + 4, std::numeric_limits<float>::quiet_NaN());
  CB_TRY(h.ev.create());
  Events& ev = h.ev;
  ScopedEvents total;
  CB_TRY(total.create());
  DeviceScope scope(ctx);
  CB_TRY(scope.alloc(&h.d_idx, 3 * (size_t)kMaxBatch));
  CB_TRY(scope.alloc(&h.d_planes, kMaxBatch));
  CB_TRY(scope.alloc(&h.d_counts, kMaxBatch));
  CB_CUDA(cudaEventRecord(total.e0, ctx->stream));
  RansacRun run;
  CB_TRY(ransac_loop(sampler, inlier_count_thresh, max_iter, kFirstBatch, kMaxBatch, h, &run));
  // No hypothesis ever reached sample_size inliers: the reference's model is an uninitialised Eigen::Hyperplane;
  // NaN stands in for it, with or without re-estimation.
  float plane[4];
  std::memcpy(plane, h.best, sizeof(plane));
  double ms_re = 0.0;
  if (re_estimate && run.have_best) {  // :118-120
    CB_CUDA(cudaEventRecord(ev.e[3], ctx->stream));
    CB_TRY(reestimate(ctx, cloud, h.best, thresh, run.best_count, plane));
    CB_CUDA(cudaEventRecord(ev.e[4], ctx->stream));
    CB_CUDA(cudaEventSynchronize(ev.e[4]));
    ms_re = ev.ms(3, 4);
  }
  // the model's residuals and inliers (:95-101 for the kept hypothesis, :121-127 after re-estimation)
  size_t n_inl = 0;
  CB_CUDA(cudaEventRecord(ev.e[3], ctx->stream));
  CB_TRY(cb_plane_residuals(ctx, cloud, plane, thresh, residuals, inliers, &n_inl));
  CB_CUDA(cudaEventRecord(ev.e[4], ctx->stream));
  CB_CUDA(cudaEventRecord(total.e1, ctx->stream));
  CB_CUDA(cudaEventSynchronize(total.e1));
  float ms = 0.f;
  CB_CUDA(cudaEventElapsedTime(&ms, total.e0, total.e1));
  std::memcpy(res->plane, plane, sizeof(plane));
  std::memcpy(res->hyp_plane, h.best, sizeof(h.best));
  res->iterations = run.iterations;
  res->best_iteration = run.best_iteration;
  res->num_inliers = n_inl;
  res->gpu_ms_total = ms;
  res->gpu_ms_fit = h.ms_fit;
  res->gpu_ms_score = h.ms_score;
  res->gpu_ms_reestimate = ms_re;
  res->gpu_ms_final = ev.ms(3, 4);
  res->kernel_launches = ctx->launches - launches0;
  return CB_OK;
}

}  // extern "C"
