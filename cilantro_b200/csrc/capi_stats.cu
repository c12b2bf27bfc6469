// C ABI: covariance / PCA (product code).
#include "cb_internal.hpp"
#include "stats_kernels.cuh"
#include "host_solve.hpp"
#include <cmath>
#include <cstring>
#include <limits>
#include <vector>

using namespace cb;

// Mean and (n-1)-normalised covariance. The reference does two serial passes (mean, then centred
// outer products, core/covariance.hpp:64-76); here: a tiny first launch over <= 4096 points gives a
// pivot close to the mean, then ONE streaming pass accumulates sum(p - c) and sum (p - c)(p - c)^T in
// double, which is combined exactly: cov = (S2 - S1 S1^T / n) / (n - 1), mean = c + S1 / n.
static int mean_cov_double(cb_context* ctx, const float* raw, size_t npts, double* mean3, double* cov9, double* n_out) {
  CB_CUDA(cudaSetDevice(ctx->device));
  const float zero[3] = {0, 0, 0};
  double m[kMomentValues];
  float pivot[3] = {0, 0, 0};
  if (npts > 0) {
    const size_t head = npts < 4096 ? npts : 4096;
    CB_TRY(launch_moments(ctx, raw, head, zero));
    CB_TRY(fetch_result(ctx, kMomentValues, false, m));
    for (int r = 0; r < 3; r++) pivot[r] = (float)(m[1 + r] / m[0]);
  }
  if (ctx->world > 1) {
    // every rank must use the same pivot: average the non-empty ranks' pivots (4-value all-reduce)
    const double wgt = npts > 0 ? 1.0 : 0.0;
    double pv[4] = {pivot[0] * wgt, pivot[1] * wgt, pivot[2] * wgt, wgt};
    std::memcpy(ctx->h_result, pv, sizeof(pv));
    CB_CUDA(cudaMemcpyAsync(ctx->d_result, ctx->h_result, sizeof(pv), cudaMemcpyHostToDevice, ctx->stream));
    CB_TRY(fetch_result(ctx, 4, true, pv));
    for (int r = 0; r < 3; r++) pivot[r] = pv[3] > 0 ? (float)(pv[r] / pv[3]) : 0.f;
  }
  CB_TRY(launch_moments(ctx, raw, npts, pivot));
  CB_TRY(fetch_result(ctx, kMomentValues, true, m));
  const double n = m[0];
  *n_out = n;
  if (n < 2.0) return CB_OK;
  const double s1[3] = {m[1], m[2], m[3]};
  const double s2[3][3] = {{m[4], m[5], m[6]}, {m[5], m[7], m[8]}, {m[6], m[8], m[9]}};
  for (int r = 0; r < 3; r++) mean3[r] = (double)pivot[r] + s1[r] / n;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) cov9[r * 3 + c] = (s2[r][c] - s1[r] * s1[c] / n) / (n - 1.0);
  return CB_OK;
}

extern "C" {

int cb_mean_cov(cb_context* ctx, const cb_cloud* pts, float* mean3, float* cov9) {
  CB_CHECK(ctx && pts && mean3 && cov9, CB_ERR_INVALID, "null argument");
  double mu[3], cov[9], n = 0;
  CB_TRY(mean_cov_double(ctx, pts->d_raw, pts->n, mu, cov, &n));
  if (n < 2.0) {  // covariance.hpp:35-38 (min_sample_size_ = 2)
    for (int i = 0; i < 3; i++) mean3[i] = std::numeric_limits<float>::quiet_NaN();
    for (int i = 0; i < 9; i++) cov9[i] = std::numeric_limits<float>::quiet_NaN();
    return 0;
  }
  for (int i = 0; i < 3; i++) mean3[i] = (float)mu[i];
  for (int i = 0; i < 9; i++) cov9[i] = (float)cov[i];
  return 1;
}

int cb_pca(cb_context* ctx, const cb_cloud* pts, float* mean3, float* cov9, float* evals3, float* evecs9) {
  CB_CHECK(ctx && pts && mean3 && cov9 && evals3 && evecs9, CB_ERR_INVALID, "null argument");
  double mu[3], cov[9], n = 0;
  CB_TRY(mean_cov_double(ctx, pts->d_raw, pts->n, mu, cov, &n));
  if (n < 2.0) {
    for (int i = 0; i < 3; i++) mean3[i] = evals3[i] = std::numeric_limits<float>::quiet_NaN();
    for (int i = 0; i < 9; i++) cov9[i] = evecs9[i] = std::numeric_limits<float>::quiet_NaN();
    return 0;
  }
  for (int i = 0; i < 3; i++) mean3[i] = (float)mu[i];
  double covf[9];
  for (int i = 0; i < 9; i++) {
    cov9[i] = (float)cov[i];
    covf[i] = (double)cov9[i];  // the eigen-solver sees the fp32 covariance, as in the reference (:77)
  }
  pca_from_cov(covf, evals3, evecs9);
  return 1;
}

}  // extern "C"

// ---- D-dimensional vector sets ----------------------------------------------------------------------------------
// Covariance<float, D>::operator() over the whole set (subset == NULL) or the listed rows (covariance.hpp:30-179). The
// sample-size rule and the n = 0 / n = 1 expressions of the reference are settled here, before any kernel runs;
// n >= 2 runs the moments kernel at D = 3 (the bits of cb_mean_cov) and pca_features.cu otherwise.
static int vectors_mean_cov(cb_context* ctx, const cb_vectors* v, const uint64_t* subset, size_t m,
                            size_t min_sample_size, float* mean, float* cov) {
  CB_CHECK(ctx && v && mean && cov, CB_ERR_INVALID, "null argument");
  CB_CHECK(v->ctx == ctx, CB_ERR_INVALID, "vector set belongs to another context");
  CB_CHECK(ctx->world == 1, CB_ERR_UNSUPPORTED, "covariance over vector sets runs on one GPU");
  const int D = v->D;
  const size_t DD = (size_t)D * D;
  const size_t n = subset ? m : v->n;
  for (size_t i = 0; subset && i < m; i++) CB_CHECK(subset[i] < v->n, CB_ERR_INVALID, "subset index out of range");
  const float nan = std::numeric_limits<float>::quiet_NaN();
  if (n < min_sample_size) {  // covariance.hpp:35-38
    std::fill(mean, mean + D, nan);
    std::fill(cov, cov + DD, nan);
    return 0;
  }
  if (n == 0) {
    // mean = (1 / 0) * 0; cov = (1 / (n - 1)) * 0 with n - 1 = -1 as an Eigen::Index (whole set, -0) or 2^64 - 1 as a
    // size_t (subset overloads, +0)
    std::fill(mean, mean + D, nan);
    std::fill(cov, cov + DD, subset ? 0.f : -0.f);
    return 1;
  }
  CB_CUDA(cudaSetDevice(ctx->device));
  if (n == 1) {  // mean = the row, cov = (1 / 0) * 0
    const size_t row = subset ? subset[0] : 0;
    CB_CUDA(cudaMemcpyAsync(mean, v->d_raw + row * (size_t)D, (size_t)D * sizeof(float), cudaMemcpyDeviceToHost,
                            ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    std::fill(cov, cov + DD, nan);
    return 1;
  }
  DeviceScope scope(ctx);
  const float* rows = v->d_raw;
  if (subset) {  // gathered into scratch: the result is the whole-set result of the gathered rows
    uint64_t* d_idx = nullptr;
    float* d_rows = nullptr;
    CB_TRY(scope.alloc(&d_idx, m));
    CB_TRY(scope.alloc(&d_rows, m * (size_t)D));
    CB_CUDA(cudaMemcpyAsync(d_idx, subset, m * sizeof(uint64_t), cudaMemcpyHostToDevice, ctx->stream));
    CB_TRY(vectors_gather(ctx, v->d_raw, D, d_idx, m, d_rows));
    rows = d_rows;
  }
  if (D != 3) {
    CB_TRY(features_mean_cov(ctx, rows, n, D, mean, cov));
    return 1;
  }
  double mu[3], c9[9], nn = 0;
  CB_TRY(mean_cov_double(ctx, rows, n, mu, c9, &nn));
  for (int i = 0; i < 3; i++) mean[i] = (float)mu[i];
  for (int i = 0; i < 9; i++) cov[i] = (float)c9[i];
  return 1;
}

extern "C" {

int cb_vectors_mean_cov(cb_context* ctx, const cb_vectors* v, const uint64_t* subset, size_t m,
                        size_t min_sample_size, float* mean, float* cov) {
  return vectors_mean_cov(ctx, v, subset, m, min_sample_size, mean, cov);
}

int cb_vectors_pca(cb_context* ctx, const cb_vectors* v, const uint64_t* subset, size_t m, size_t min_sample_size,
                   float* mean, float* cov, float* evals, float* evecs) {
  CB_CHECK(evals && evecs, CB_ERR_INVALID, "null argument");
  const int rc = vectors_mean_cov(ctx, v, subset, m, min_sample_size, mean, cov);
  if (rc < 0) return rc;
  const int D = v->D;
  const size_t DD = (size_t)D * D;
  if (rc == 0) {
    std::fill(evals, evals + D, std::numeric_limits<float>::quiet_NaN());
    std::fill(evecs, evecs + DD, std::numeric_limits<float>::quiet_NaN());
    return 0;
  }
  std::vector<double> covf(DD);  // the eigen-solver sees the fp32 covariance (principal_component_analysis.hpp:77)
  for (size_t i = 0; i < DD; i++) covf[i] = (double)cov[i];
  if (D == 3) {
    pca_from_cov(covf.data(), evals, evecs);
    return 1;
  }
  CB_CHECK(sym_eigen(covf.data(), D, evals, evecs) >= 0, CB_ERR_UNSUPPORTED,
           "PCA: the symmetric QR iteration did not converge");
  return 1;
}

}  // extern "C"

// PrincipalComponentAnalysis::project / reconstruct (principal_component_analysis.hpp:46-68) with the first k columns
// of evecs: x (n x din) -> n x dout, on the device, to the host and / or into a new vector set.
static int vectors_map(cb_context* ctx, const cb_vectors* x, const float* mean, const float* evecs, int D, int k,
                       bool project, float* out_host, cb_vectors** out_device) {
  CB_CHECK(ctx && x && mean && evecs, CB_ERR_INVALID, "null argument");
  CB_CHECK(out_host || out_device, CB_ERR_INVALID, "no output requested");
  CB_CHECK(x->ctx == ctx, CB_ERR_INVALID, "vector set belongs to another context");
  CB_CHECK(ctx->world == 1, CB_ERR_UNSUPPORTED, "PCA projection over vector sets runs on one GPU");
  CB_CHECK(k >= 1 && k <= D, CB_ERR_INVALID, "k must be in [1, D]");
  CB_CHECK(x->D == (project ? D : k), CB_ERR_INVALID, "dimension mismatch");
  if (out_device) *out_device = nullptr;
  CB_CUDA(cudaSetDevice(ctx->device));
  const int din = project ? D : k, dout = project ? k : D;
  const size_t n = x->n;
  cb_vectors* res = new cb_vectors(ctx, n, dout);
  auto run = [&]() -> int {
    DeviceScope scope(ctx);
    float *d_E = nullptr, *d_mean = nullptr;
    CB_TRY(scope.alloc(&d_E, (size_t)D * D));
    CB_TRY(scope.alloc(&d_mean, (size_t)D));
    CB_CUDA(cudaMemcpyAsync(d_E, evecs, (size_t)D * D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    CB_CUDA(cudaMemcpyAsync(d_mean, mean, (size_t)D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    CB_TRY(res->mem.alloc(&res->d_raw, n * (size_t)dout));
    if (n) {
      if (project)
        CB_TRY(features_map(ctx, x->d_raw, n, D, k, d_E, D, 1, d_mean, true, res->d_raw));
      else
        CB_TRY(features_map(ctx, x->d_raw, n, k, D, d_E, 1, D, d_mean, false, res->d_raw));
      if (out_host)
        CB_CUDA(cudaMemcpyAsync(out_host, res->d_raw, n * (size_t)dout * sizeof(float), cudaMemcpyDeviceToHost,
                                ctx->stream));
    }
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    return CB_OK;
  };
  const int rc = run();
  if (rc != CB_OK || !out_device) {
    delete res;
    return rc;
  }
  *out_device = res;
  return CB_OK;
}

extern "C" {

int cb_vectors_project(cb_context* ctx, const cb_vectors* v, const float* mean, const float* evecs, int k,
                       float* out_host, cb_vectors** out_device) {
  CB_CHECK(v, CB_ERR_INVALID, "null argument");
  return vectors_map(ctx, v, mean, evecs, v->D, k, true, out_host, out_device);
}

int cb_vectors_reconstruct(cb_context* ctx, const cb_vectors* q, const float* mean, const float* evecs, int D,
                           float* out_host, cb_vectors** out_device) {
  CB_CHECK(q, CB_ERR_INVALID, "null argument");
  return vectors_map(ctx, q, mean, evecs, D, q->D, false, out_host, out_device);
}

}  // extern "C"
