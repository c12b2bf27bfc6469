// RANSAC hypothesis scoring for rigid transforms (product code, sm_90a).
//
// Replaces, for H hypotheses at once, TransformRANSACEstimator::computeResiduals
// (model_estimation/ransac_transform_estimator.hpp:90-98) followed by the serial inlier scan of
// RandomSampleConsensusBase::estimate (model_estimation/ransac_base.hpp:96-101):
//   residual_i = |T s_i - d_i|  (fp32, contract arithmetic below), inlier iff residual_i <= thresh.
// The reference streams the 2 x 12 B x N pairs from DRAM once PER hypothesis and writes a 4 B x N
// residual vector each time; here a tile of pairs sits in registers while ALL hypotheses of the
// batch (staged in shared memory, broadcast to the warp) are scored against it, so the pairs are
// read once per batch and only H integers leave the chip. Bound: FP32 pipe (~28 instr / pair-hyp).
//
// Arithmetic contract (oracle/cilantro_oracle.cpp): q_r = (R_r0 x + (R_r1 y + R_r2 z)) + t_r,
// e = q - d, x = e0^2 + (e1^2 + e2^2), residual = sqrt_rn(x). The comparison sqrt_rn(x) <= thresh is
// evaluated as x <= x_max with x_max = max{x : sqrt_rn(x) <= thresh} found on the host (sqrt_rn is
// monotone), which is bit-equivalent and keeps the MUFU pipe out of the inner loop.
#include "cb_internal.hpp"
#include "nn_search.cuh"
#include "reduce.cuh"
#include "host_solve.hpp"
#include "ransac_sampler.hpp"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

using namespace cb;

namespace {

constexpr int kBlock = 256;
constexpr int kPairs = 4;        // pairs per thread in registers
constexpr int kHypChunk = 256;   // hypotheses staged in shared memory at a time
constexpr int kMaxBatch = 16384; // hypotheses per launch (shared-memory vote counters)

__global__ void __launch_bounds__(kBlock) ransac_score_kernel(const float* __restrict__ dst, const float* __restrict__ src,
                                                              size_t n, const float* __restrict__ T_h, int H,
                                                              float x_max, uint32_t* __restrict__ counts) {
  extern __shared__ unsigned char smem_raw[];
  float* s_T = reinterpret_cast<float*>(smem_raw);                                            // kHypChunk * 12
  uint32_t* s_cnt = reinterpret_cast<uint32_t*>(smem_raw + (size_t)kHypChunk * 12 * sizeof(float));  // H
  for (int h = threadIdx.x; h < H; h += kBlock) s_cnt[h] = 0;
  const size_t tile = (size_t)kBlock * kPairs;
  const int lane = threadIdx.x & 31;
  for (size_t base = (size_t)blockIdx.x * tile; base < n; base += (size_t)gridDim.x * tile) {
    float sx[kPairs], sy[kPairs], sz[kPairs], dx[kPairs], dy[kPairs], dz[kPairs];
    bool ok[kPairs];
#pragma unroll
    for (int u = 0; u < kPairs; u++) {
      const size_t i = base + (size_t)u * kBlock + threadIdx.x;
      ok[u] = i < n;
      sx[u] = ok[u] ? src[3 * i] : 0.f;
      sy[u] = ok[u] ? src[3 * i + 1] : 0.f;
      sz[u] = ok[u] ? src[3 * i + 2] : 0.f;
      dx[u] = ok[u] ? dst[3 * i] : 0.f;
      dy[u] = ok[u] ? dst[3 * i + 1] : 0.f;
      dz[u] = ok[u] ? dst[3 * i + 2] : 0.f;
    }
    for (int h0 = 0; h0 < H; h0 += kHypChunk) {
      const int hn = min(kHypChunk, H - h0);
      __syncthreads();
      for (int j = threadIdx.x; j < hn * 12; j += kBlock) s_T[j] = T_h[(size_t)h0 * 12 + j];
      __syncthreads();
      for (int h = 0; h < hn; h++) {
        const float4 r0 = *reinterpret_cast<const float4*>(s_T + h * 12);
        const float4 r1 = *reinterpret_cast<const float4*>(s_T + h * 12 + 4);
        const float4 r2 = *reinterpret_cast<const float4*>(s_T + h * 12 + 8);
        int c = 0;
#pragma unroll
        for (int u = 0; u < kPairs; u++) {
          const float qx = __fadd_rn(sum3(__fmul_rn(r0.x, sx[u]), __fmul_rn(r0.y, sy[u]), __fmul_rn(r0.z, sz[u])), r0.w);
          const float qy = __fadd_rn(sum3(__fmul_rn(r1.x, sx[u]), __fmul_rn(r1.y, sy[u]), __fmul_rn(r1.z, sz[u])), r1.w);
          const float qz = __fadd_rn(sum3(__fmul_rn(r2.x, sx[u]), __fmul_rn(r2.y, sy[u]), __fmul_rn(r2.z, sz[u])), r2.w);
          const float e0 = __fsub_rn(qx, dx[u]), e1 = __fsub_rn(qy, dy[u]), e2 = __fsub_rn(qz, dz[u]);
          const float x = sum3(__fmul_rn(e0, e0), __fmul_rn(e1, e1), __fmul_rn(e2, e2));
          c += (ok[u] && x <= x_max) ? 1 : 0;
        }
        c = __reduce_add_sync(0xffffffffu, c);
        if (lane == 0 && c) atomicAdd(s_cnt + h0 + h, (uint32_t)c);
      }
    }
  }
  __syncthreads();
  for (int h = threadIdx.x; h < H; h += kBlock)
    if (s_cnt[h]) atomicAdd(counts + h, s_cnt[h]);
}

// residuals of one model, with the real (correctly rounded) square root
__global__ void ransac_residual_kernel(const float* __restrict__ dst, const float* __restrict__ src, size_t n,
                                       const Rigid T, float* __restrict__ out) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float qx, qy, qz;
    rule::transform_point(T, src[3 * i], src[3 * i + 1], src[3 * i + 2], qx, qy, qz);
    const float e0 = __fsub_rn(qx, dst[3 * i]), e1 = __fsub_rn(qy, dst[3 * i + 1]), e2 = __fsub_rn(qz, dst[3 * i + 2]);
    out[i] = __fsqrt_rn(sum3(__fmul_rn(e0, e0), __fmul_rn(e1, e1), __fmul_rn(e2, e2)));
  }
}

// Kabsch moments over the inliers of model T (re-estimation step, ransac_base.hpp:118-120):
// {n, sum d (3), sum s (3), sum d s^T (9)} over pairs with residual <= thresh.
__global__ void __launch_bounds__(kReduceBlock) inlier_moments_kernel(const float* __restrict__ dst,
                                                                      const float* __restrict__ src, size_t n,
                                                                      const Rigid T, float x_max, const ReduceScratch rs) {
  double acc[16];
#pragma unroll
  for (int i = 0; i < 16; i++) acc[i] = 0.0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float s0 = src[3 * i], s1 = src[3 * i + 1], s2 = src[3 * i + 2];
    const float d0 = dst[3 * i], d1 = dst[3 * i + 1], d2 = dst[3 * i + 2];
    float qx, qy, qz;
    rule::transform_point(T, s0, s1, s2, qx, qy, qz);
    const float e0 = __fsub_rn(qx, d0), e1 = __fsub_rn(qy, d1), e2 = __fsub_rn(qz, d2);
    const float x = sum3(__fmul_rn(e0, e0), __fmul_rn(e1, e1), __fmul_rn(e2, e2));
    if (!(x <= x_max)) continue;
    const double D0 = d0, D1 = d1, D2 = d2, S0 = s0, S1 = s1, S2 = s2;
    acc[0] += 1.0;
    acc[1] += D0; acc[2] += D1; acc[3] += D2;
    acc[4] += S0; acc[5] += S1; acc[6] += S2;
    acc[7] += D0 * S0;  acc[8] += D0 * S1;  acc[9] += D0 * S2;
    acc[10] += D1 * S0; acc[11] += D1 * S1; acc[12] += D1 * S2;
    acc[13] += D2 * S0; acc[14] += D2 * S1; acc[15] += D2 * S2;
  }
  grid_reduce<16>(acc, rs);
}

__global__ void gather_pairs_kernel(const float* __restrict__ dst, const float* __restrict__ src,
                                    const uint32_t* __restrict__ idx, size_t m, float* __restrict__ out) {
  for (size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x; k < m; k += (size_t)gridDim.x * blockDim.x) {
    const size_t i = idx[k];
#pragma unroll
    for (int r = 0; r < 3; r++) {
      out[6 * k + r] = dst[3 * i + r];
      out[6 * k + 3 + r] = src[3 * i + r];
    }
  }
}

__global__ void u32_to_f64_kernel(const uint32_t* __restrict__ in, double* __restrict__ out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (double)in[i];
}
__global__ void f64_to_u32_kernel(const double* __restrict__ in, uint32_t* __restrict__ out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (uint32_t)(in[i] + 0.5);
}

// largest x with sqrt_rn(x) <= thresh
float sqrt_threshold(float thresh) {
  if (!(thresh >= 0.f)) return -1.0f;           // negative or NaN threshold: nothing is an inlier
  if (std::isinf(thresh)) return thresh;
  float x = thresh * thresh;
  while (std::sqrt(x) <= thresh) {
    float nx = std::nextafter(x, INFINITY);
    if (std::isinf(nx) || !(std::sqrt(nx) <= thresh)) break;
    x = nx;
  }
  while (std::sqrt(x) > thresh) x = std::nextafter(x, -INFINITY);
  return x;
}

int check_pair(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src) {
  CB_CHECK(ctx && dst && src, CB_ERR_INVALID, "null argument");
  CB_CHECK(dst->ctx == ctx && src->ctx == ctx, CB_ERR_INVALID, "cloud belongs to another context");
  CB_CHECK(dst->n == src->n, CB_ERR_INVALID, "dst and src must be paired (equal size)");
  CB_CUDA(cudaSetDevice(ctx->device));
  return CB_OK;
}

// scores H <= kMaxBatch hypotheses already in device memory; counts (device, H) zeroed here
int score_batch(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src, const float* d_T, int H, float x_max,
                uint32_t* d_counts) {
  CB_CUDA(cudaMemsetAsync(d_counts, 0, (size_t)H * sizeof(uint32_t), ctx->stream));
  if (dst->n == 0 || H == 0) return CB_OK;
  const size_t smem = (size_t)kHypChunk * 12 * sizeof(float) + (size_t)H * sizeof(uint32_t);
  CB_CUDA(cudaFuncSetAttribute(ransac_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const size_t tile = (size_t)kBlock * kPairs;
  int per_sm = 0;  // resident blocks per SM for this launch's dynamic shared memory (a fixed 2 left most warp slots empty)
  CB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ransac_score_kernel, kBlock, smem));
  per_sm = std::max(1, std::min(per_sm, 6));
  const int blocks = (int)std::max<size_t>(1, std::min<size_t>((size_t)ctx->sm_count * per_sm, (dst->n + tile - 1) / tile));
  ransac_score_kernel<<<blocks, kBlock, smem, ctx->stream>>>(dst->d_raw, src->d_raw, dst->n, d_T, H, x_max, d_counts);
  ctx->launches += 1;
  CB_CUDA(cudaGetLastError());
  if (ctx->world > 1) {
    DeviceScope scope(ctx);
    double* d_tmp = nullptr;
    CB_TRY(scope.alloc(&d_tmp, (size_t)H));
    u32_to_f64_kernel<<<(H + 255) / 256, 256, 0, ctx->stream>>>(d_counts, d_tmp, H);
    CB_TRY(nccl_allreduce_sum_f64(ctx, d_tmp, (size_t)H));
    f64_to_u32_kernel<<<(H + 255) / 256, 256, 0, ctx->stream>>>(d_tmp, d_counts, H);
    ctx->launches += 2;
  }
  return CB_OK;
}

Rigid rigid_of(const float* T12) {
  Rigid r;
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) r.r[i * 3 + j] = T12[i * 4 + j];
    r.t[i] = T12[i * 4 + 3];
  }
  return r;
}

int residuals_device(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src, const float* T12, float* d_out) {
  if (dst->n == 0) return CB_OK;
  const int blocks = (int)std::max<size_t>(1, std::min<size_t>((size_t)ctx->sm_count * 8, (dst->n + 255) / 256));
  ransac_residual_kernel<<<blocks, 256, 0, ctx->stream>>>(dst->d_raw, src->d_raw, dst->n, rigid_of(T12), d_out);
  ctx->launches += 1;
  CB_CUDA(cudaGetLastError());
  return CB_OK;
}

}  // namespace

extern "C" {

int cb_ransac_score(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src, const float* T_h, size_t H,
                    float thresh, uint32_t* counts) {
  CB_TRY(check_pair(ctx, dst, src));
  CB_CHECK(H == 0 || (T_h && counts), CB_ERR_INVALID, "null argument");
  const float x_max = sqrt_threshold(thresh);
  DeviceScope scope(ctx);
  float* d_T = nullptr;
  uint32_t* d_counts = nullptr;
  const size_t cap = std::min<size_t>(H, kMaxBatch);
  CB_TRY(scope.alloc(&d_T, cap * 12));
  CB_TRY(scope.alloc(&d_counts, cap));
  for (size_t h0 = 0; h0 < H; h0 += kMaxBatch) {
    const int hn = (int)std::min<size_t>(kMaxBatch, H - h0);
    CB_CUDA(cudaMemcpyAsync(d_T, T_h + 12 * h0, (size_t)hn * 12 * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    CB_TRY(score_batch(ctx, dst, src, d_T, hn, x_max, d_counts));
    CB_CUDA(cudaMemcpyAsync(counts + h0, d_counts, (size_t)hn * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  return CB_OK;
}

int cb_ransac_residuals(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src, const float* T12, float thresh,
                        float* residuals, uint64_t* inliers, size_t* num_inliers) {
  CB_TRY(check_pair(ctx, dst, src));
  CB_CHECK(T12, CB_ERR_INVALID, "null argument");
  const size_t n = dst->n;
  std::vector<float> h(n);
  if (n) {
    DeviceScope scope(ctx);
    float* d_out = nullptr;
    CB_TRY(scope.alloc(&d_out, n));
    CB_TRY(residuals_device(ctx, dst, src, T12, d_out));
    CB_CUDA(cudaMemcpyAsync(h.data(), d_out, n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  size_t k = 0;
  for (size_t i = 0; i < n; i++) {
    if (residuals) residuals[i] = h[i];
    if (h[i] <= thresh) {  // ransac_base.hpp:99
      if (inliers) inliers[k] = (uint64_t)i + dst->index_offset;
      ++k;
    }
  }
  if (num_inliers) *num_inliers = k;
  return CB_OK;
}

int cb_ransac_rigid(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src, uint32_t seed,
                    size_t inlier_count_thresh, size_t max_iter, float thresh, int re_estimate,
                    cb_ransac_result* res, uint64_t* inliers, float* residuals) {
  CB_TRY(check_pair(ctx, dst, src));
  CB_CHECK(res, CB_ERR_INVALID, "null argument");
  CB_CHECK(ctx->world == 1, CB_ERR_UNSUPPORTED, "cb_ransac_rigid runs per process; shard hypotheses with cb_ransac_score");
  const uint64_t launches0 = ctx->launches;
  const size_t n = dst->n;
  size_t sample_size = 3;  // MinSampleSize for a rigid 3-D transform (ransac_transform_estimator.hpp:21-23)
  if (n < sample_size) sample_size = n;                   // ransac_base.hpp:67
  if (inlier_count_thresh > n) inlier_count_thresh = n;   // :68
  const float x_max = sqrt_threshold(thresh);

  RansacSampler sampler(n, seed);  // :72-73 with the seed injected

  float best_T[12];
  t34_identity(best_T);
  size_t best_count = 0, best_it = 0, it = 0;
  bool have_best = false, done = false;

  const size_t B = 1024;  // hypotheses generated and scored per round trip
  DeviceScope scope(ctx);
  float* d_T = nullptr;
  uint32_t* d_counts = nullptr;
  uint32_t* d_idx = nullptr;
  float* d_pairs = nullptr;
  CB_TRY(scope.alloc(&d_T, B * 12));
  CB_TRY(scope.alloc(&d_counts, B));
  CB_TRY(scope.alloc(&d_idx, B * 3));
  CB_TRY(scope.alloc(&d_pairs, B * 3 * 6));
  std::vector<uint32_t> h_idx(B * 3), h_counts(B);
  std::vector<float> h_pairs(B * 18), h_T(B * 12);
  ScopedEvents ev;
  CB_TRY(ev.create());
  CB_CUDA(cudaEventRecord(ev.e0, ctx->stream));
  while (!done && it < max_iter) {
    const size_t nb = std::min(B, max_iter - it);
    // sample (:83-91): partial Fisher-Yates on a permutation that persists across hypotheses
    for (size_t b = 0; b < nb; b++) sampler.next(sample_size, &h_idx[b * 3]);
    // estimateModel(sample) (:94, ransac_transform_estimator.hpp:72-82): Kabsch on the sample
    if (sample_size > 0) {
      CB_CUDA(cudaMemcpyAsync(d_idx, h_idx.data(), nb * 3 * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
      gather_pairs_kernel<<<(int)((nb * 3 + 255) / 256), 256, 0, ctx->stream>>>(dst->d_raw, src->d_raw, d_idx, nb * 3,
                                                                              d_pairs);
      ctx->launches += 1;
      CB_CUDA(cudaMemcpyAsync(h_pairs.data(), d_pairs, nb * 18 * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
      CB_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    for (size_t b = 0; b < nb; b++) {
      double m[16] = {0};
      for (size_t i = 0; i < sample_size; i++) {
        const float* p = &h_pairs[(b * 3 + i) * 6];
        m[0] += 1.0;
        for (int r = 0; r < 3; r++) {
          m[1 + r] += p[r];
          m[4 + r] += p[3 + r];
          for (int c = 0; c < 3; c++) m[7 + r * 3 + c] += (double)p[r] * (double)p[3 + c];
        }
      }
      kabsch_from_moments(m, &h_T[b * 12]);
    }
    CB_CUDA(cudaMemcpyAsync(d_T, h_T.data(), nb * 12 * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    CB_TRY(score_batch(ctx, dst, src, d_T, (int)nb, x_max, d_counts));
    CB_CUDA(cudaMemcpyAsync(h_counts.data(), d_counts, nb * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    // sequential semantics over the batch (:103-114)
    for (size_t b = 0; b < nb; b++) {
      it++;
      const size_t cnt = h_counts[b];
      if (cnt < sample_size) continue;       // :104
      if (cnt > best_count) {                // :107 (model_inliers_ starts empty, so size 0)
        best_count = cnt;
        std::memcpy(best_T, &h_T[b * 12], sizeof(best_T));
        best_it = it - 1;
        have_best = true;
      }
      if (best_count >= inlier_count_thresh) {  // :114
        done = true;
        break;
      }
    }
  }
  // no hypothesis ever reached sample_size inliers: model_inliers_ is empty, so the re-estimation
  // is a Kabsch over zero pairs = identity (transform_estimation.hpp:20-23)
  if (re_estimate && have_best) {  // :118-128
    const int blocks = (int)std::max<size_t>(1, std::min<size_t>((size_t)ctx->sm_count * 4, (n + kReduceBlock - 1) / kReduceBlock));
    ReduceScratch rs;
    CB_TRY(get_reduce_scratch(ctx, blocks, 16, &rs));
    inlier_moments_kernel<<<blocks, kReduceBlock, 0, ctx->stream>>>(dst->d_raw, src->d_raw, n, rigid_of(best_T), x_max, rs);
    ctx->launches += 1;
    double m[16];
    CB_CUDA(cudaMemcpyAsync(ctx->h_result, ctx->d_result, sizeof(m), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    std::memcpy(m, ctx->h_result, sizeof(m));
    kabsch_from_moments(m, best_T);
  }
  size_t n_inl = best_count;
  CB_CUDA(cudaEventRecord(ev.e1, ctx->stream));
  CB_TRY(cb_ransac_residuals(ctx, dst, src, best_T, thresh, residuals, inliers, &n_inl));
  CB_CUDA(cudaEventSynchronize(ev.e1));  // (cb_ransac_residuals does not synchronise an empty cloud)
  float ms = 0.f;
  CB_CUDA(cudaEventElapsedTime(&ms, ev.e0, ev.e1));
  std::memcpy(res->T, best_T, sizeof(best_T));
  res->iterations = it;
  res->num_inliers = n_inl;
  res->best_iteration = best_it;
  res->gpu_ms_total = ms;
  res->kernel_launches = ctx->launches - launches0;
  return CB_OK;
}

}  // extern "C"
