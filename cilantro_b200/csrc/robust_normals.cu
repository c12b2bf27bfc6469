// Robust per-point normal estimation (product code, sm_90a): NormalEstimation<float, 3,
// MinimumCovarianceDeterminant<float, 3>> (core/normal_estimation.hpp:279-421 over core/covariance.hpp:185-371) for
// kNN and kNN-in-radius neighbourhoods of at most 128 points. Two kernels (DESIGN §4.15):
//   * mcd_search_kernel: one thread per point of the cell-sorted cloud finds its k best (d2, original index) pairs
//     over the grid, with the admission and order of normals_knn_kernel, and writes the original indices;
//   * mcd_kernel: one warp per point stages the neighbourhood's coordinates in shared memory and runs the trials.
//     The serial parts (draws, h-sums, determinant, chi-square test) run on every lane alike, so their results need
//     no broadcast; the Mahalanobis keys are computed four per lane and the kept subset is found by ranking the
//     packed (key, position) values, each lane counting the smaller ones for its own four.
// The arithmetic, the generator and the selection order are those of mcd_rule.hpp; the eigen solve and the
// orientation step are the plain path's (normals_out.cuh).
#include "cb_internal.hpp"
#include "grid_sweep.cuh"
#include "kbest.cuh"
#include "launch.cuh"
#include "mcd_rule.hpp"
#include "normals_out.cuh"
#include <algorithm>
#include <cfloat>
#include <cmath>

using namespace cb;

namespace {

constexpr int kBlock = 128;
constexpr int kWarps = kBlock / 32;
constexpr int kPerLane = mcd::kMaxK / 32;

struct McdArgs {
  uint32_t trials, refinements, min_size;
  float ratio, chi2;
  uint32_t seed;
};

template <int K>
__global__ void __launch_bounds__(kBlock) mcd_search_kernel(const GridView g, int k, float max_d2,
                                                            int* __restrict__ nbr, uint8_t* __restrict__ cnt) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t qi = blockIdx.x * blockDim.x + threadIdx.x; qi < g.n; qi += stride) {
    const float4 s = __ldg(g.pts + qi);
    float bd[K];
    int bi[K];
    int count = 0;
    auto bound = [&]() { return (count == k) ? bd[k - 1] : max_d2; };
    auto scan = [&](uint32_t b, uint32_t e) {
      for (uint32_t j = b; j < e; ++j) {
        const float4 p = __ldg(g.pts + j);
        const float r = rule::contract_d2(s.x, s.y, s.z, p.x, p.y, p.z);
        if (r < max_d2) kbest_insert<K>(bd, bi, k, count, r, __float_as_int(p.w));
      }
    };
    grid_sweep(g, s.x, s.y, s.z, bound, scan, [&]() { count = 0; }, (uint32_t)k);
    for (int j = 0; j < count; j++) nbr[(size_t)qi * k + j] = bi[j];
    cnt[qi] = (uint8_t)count;
  }
}

__global__ void __launch_bounds__(kBlock) mcd_kernel(const GridView g, const float* __restrict__ raw,
                                                     const int* __restrict__ nbr, const uint8_t* __restrict__ cnt, int k,
                                                     const McdArgs a, const NormalOut o, uint8_t* __restrict__ status) {
  __shared__ float sx[kWarps][mcd::kMaxK], sy[kWarps][mcd::kMaxK], sz[kWarps][mcd::kMaxK];
  __shared__ unsigned long long skey[kWarps][mcd::kMaxK];
  __shared__ uint8_t ssel[kWarps][mcd::kMaxK];
  __shared__ uint8_t sdraw[kWarps][mcd::kMaxMinSample];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t stride = gridDim.x * kWarps;
  for (uint32_t qi = blockIdx.x * kWarps + w; qi < g.n; qi += stride) {
    const float4 s = __ldg(g.pts + qi);
    const int oi = __float_as_int(s.w);
    const uint32_t m = cnt[qi];
    for (uint32_t j = lane; j < m; j += 32) {
      const size_t pi = 3 * (size_t)__ldg(nbr + (size_t)qi * k + j);
      sx[w][j] = __ldg(raw + pi);
      sy[w][j] = __ldg(raw + pi + 1);
      sz[w][j] = __ldg(raw + pi + 2);
    }
    __syncwarp();
    auto nb_at = [&](uint32_t j, float& x, float& y, float& z) {
      x = sx[w][j];
      y = sy[w][j];
      z = sz[w][j];
    };
    float mean[3], cv[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    uint8_t st = mcd::kOk;
    if (m < a.min_size) {
      st = mcd::kTooFew;
    } else if (m == a.min_size) {
      mcd::mean_cov(m, nb_at, mean, cv);  // size <= min: the plain covariance, no chi-square test (:306-307)
    } else {
      const uint32_t h = mcd::subset_size(a.ratio, m, a.min_size);
      if (h == m) {
        mcd::mean_cov(m, nb_at, mean, cv);
      } else {
        uint32_t x = mcd::minstd_seed(mcd::point_seed(a.seed, (uint32_t)oi));
        float best = FLT_MAX;
        bool found = false;
        float bmean[3], bcv[6];
        for (uint32_t t = 0; t < a.trials; t++) {
          for (uint32_t i = 0; i < a.min_size; i++) {
            const uint32_t d = mcd::uniform_below(x, m);
            if (lane == 0) sdraw[w][i] = (uint8_t)d;
          }
          __syncwarp();
          mcd::mean_cov(a.min_size, [&](uint32_t j, float& px, float& py, float& pz) { nb_at(sdraw[w][j], px, py, pz); },
                        mean, cv);
          __syncwarp();  // the next trial rewrites sdraw
          for (uint32_t r = 0; r < a.refinements; r++) {
            float inv[6];
            mcd::inverse(cv, inv);
            unsigned long long key[kPerLane];
#pragma unroll
            for (int c = 0; c < kPerLane; c++) {
              const uint32_t j = lane + 32 * c;
              key[c] = ~0ull;
              if (j < m) {
                key[c] = mcd::sort_key(mcd::mahalanobis2(inv, mcd::sub(sx[w][j], mean[0]), mcd::sub(sy[w][j], mean[1]),
                                                         mcd::sub(sz[w][j], mean[2])),
                                       j);
                skey[w][j] = key[c];
              }
            }
            __syncwarp();
            uint32_t rank[kPerLane] = {};
            for (uint32_t i = 0; i < m; i++) {
              const unsigned long long ki = skey[w][i];
#pragma unroll
              for (int c = 0; c < kPerLane; c++) rank[c] += ki < key[c];
            }
#pragma unroll
            for (int c = 0; c < kPerLane; c++)
              if (lane + 32 * c < m && rank[c] < h) ssel[w][rank[c]] = (uint8_t)(lane + 32 * c);
            __syncwarp();
            mcd::mean_cov(h, [&](uint32_t j, float& px, float& py, float& pz) { nb_at(ssel[w][j], px, py, pz); }, mean,
                          cv);
            __syncwarp();  // the next refinement rewrites skey and ssel
          }
          const float det = mcd::determinant(cv);
          if (mcd::improves(det, best)) {
            best = det;
            found = true;
#pragma unroll
            for (int c = 0; c < 3; c++) bmean[c] = mean[c];
#pragma unroll
            for (int c = 0; c < 6; c++) bcv[c] = cv[c];
          }
        }
        if (found) {
#pragma unroll
          for (int c = 0; c < 3; c++) mean[c] = bmean[c];
#pragma unroll
          for (int c = 0; c < 6; c++) cv[c] = bcv[c];
        } else {
          st = mcd::kNoFiniteTrial;
        }
      }
      if (st == mcd::kOk && a.chi2 > 0.f) {  // the neighbourhood's first point against the ellipsoid (:362-366)
        float inv[6];
        mcd::inverse(cv, inv);
        const float q =
            mcd::mahalanobis2(inv, mcd::sub(sx[w][0], mean[0]), mcd::sub(sy[w][0], mean[1]), mcd::sub(sz[w][0], mean[2]));
        if (!(q <= a.chi2)) st = mcd::kRejected;
      }
    }
    if (lane == 0) {
      finish_point(o, qi, oi, s.x, s.y, s.z, st == mcd::kOk, cv);
      if (status) status[oi] = st;
    }
    __syncwarp();  // the next point rewrites the staged coordinates
  }
}

}  // namespace

extern "C" int cb_cloud_estimate_normals_mcd(cb_context* ctx, cb_cloud* cloud, int k, float radius2,
                                             const float* view_point3, int use_current_as_ref, const cb_mcd_params* params,
                                             float* normals, float* curvature, float* cov6, uint8_t* status,
                                             float* gpu_ms) {
  CB_CHECK(ctx && cloud && params, CB_ERR_INVALID, "null argument");
  CB_CHECK(cloud->ctx == ctx, CB_ERR_INVALID, "cloud belongs to another context");
  CB_CHECK(k >= 0, CB_ERR_INVALID, "k must be >= 0");
  CB_CHECK(k > 0, CB_ERR_UNSUPPORTED, "radius-only neighbourhoods are not supported (use k > 0)");
  CB_CHECK(k <= mcd::kMaxK, CB_ERR_UNSUPPORTED, "k must be in [1, 128]");
  CB_CHECK(params->num_trials >= 1, CB_ERR_INVALID, "num_trials must be >= 1");
  CB_CHECK(params->num_refinements >= 0, CB_ERR_INVALID, "num_refinements must be >= 0");
  CB_CHECK(std::isfinite(params->inlier_ratio), CB_ERR_INVALID, "inlier_ratio must be finite");
  CB_CHECK(params->min_sample_size >= 2 && params->min_sample_size <= mcd::kMaxMinSample, CB_ERR_UNSUPPORTED,
           "min_sample_size must be in [2, 32]");
  CB_CUDA(cudaSetDevice(ctx->device));
  if (gpu_ms) *gpu_ms = 0.f;
  const size_t n = cloud->n;
  if (n == 0) return CB_OK;
  CB_TRY(ensure_index(cloud));
  const bool use_ref = use_current_as_ref && cloud->d_nrm;  // like PointCloud: only when normals exist
  if (!cloud->d_raw_nrm) CB_TRY(cloud->mem.alloc(&cloud->d_raw_nrm, 3 * n));
  if (!cloud->d_nrm) CB_TRY(cloud->mem.alloc(&cloud->d_nrm, n));
  DeviceScope scope(ctx);
  int* d_nbr = nullptr;
  uint8_t* d_cnt = nullptr;
  float* d_curv = nullptr;
  float* d_cov = nullptr;
  uint8_t* d_status = nullptr;
  CB_TRY(scope.alloc(&d_nbr, n * (size_t)k));
  CB_TRY(scope.alloc(&d_cnt, n));
  if (curvature) CB_TRY(scope.alloc(&d_curv, n));
  if (cov6) CB_TRY(scope.alloc(&d_cov, 6 * n));
  if (status) CB_TRY(scope.alloc(&d_status, n));
  NormalOut o;
  o.raw_nrm = cloud->d_raw_nrm;
  o.nrm = cloud->d_nrm;
  o.curvature = d_curv;
  o.cov6 = d_cov;
  set_orientation(o, view_point3, use_ref);
  McdArgs a;
  a.trials = (uint32_t)params->num_trials;
  a.refinements = (uint32_t)params->num_refinements;
  a.min_size = (uint32_t)params->min_sample_size;
  a.ratio = params->inlier_ratio;
  a.chi2 = params->chi_square_threshold;
  a.seed = params->seed;
  const float max_d2 = radius2 > 0.f ? radius2 : 3.402823466e38f;
  const GridView g = grid_view(cloud);
  auto search = mcd_search_kernel<128>;
  if (k <= 8)
    search = mcd_search_kernel<8>;
  else if (k <= 16)
    search = mcd_search_kernel<16>;
  else if (k <= 32)
    search = mcd_search_kernel<32>;
  else if (k <= 64)
    search = mcd_search_kernel<64>;
  ScopedEvents ev;
  if (gpu_ms) {
    CB_TRY(ev.create());
    CB_CUDA(cudaEventRecord(ev.e0, ctx->stream));
  }
  CB_TRY(launch(ctx, search, grid_for(ctx, n, kBlock), kBlock, 0, g, k, max_d2, d_nbr, d_cnt));
  CB_TRY(launch(ctx, mcd_kernel, grid_for(ctx, n, kWarps, 16), kBlock, 0, g, cloud->d_raw, d_nbr, d_cnt, k, a, o,
                d_status));
  if (gpu_ms) CB_CUDA(cudaEventRecord(ev.e1, ctx->stream));
  if (normals)
    CB_CUDA(cudaMemcpyAsync(normals, cloud->d_raw_nrm, 3 * n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  if (curvature)
    CB_CUDA(cudaMemcpyAsync(curvature, d_curv, n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  if (cov6) CB_CUDA(cudaMemcpyAsync(cov6, d_cov, 6 * n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  if (status) CB_CUDA(cudaMemcpyAsync(status, d_status, n, cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  if (gpu_ms) CB_CUDA(cudaEventElapsedTime(gpu_ms, ev.e0, ev.e1));
  return CB_OK;
}
