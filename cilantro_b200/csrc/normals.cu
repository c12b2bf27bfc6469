// Per-point normal and curvature estimation (product code, sm_90a).
// Replaces NormalEstimation::compute_normals_*/compute_normals_curvature_* (core/normal_estimation.hpp:
// 279-332, 357-421) behind PointCloud::estimateNormals{KNN,Radius,KNNInRadius} (utilities/point_cloud.hpp:
// 294-420): one thread per point of the (cell-sorted) cloud runs the neighbourhood search over the
// cloud's own grid, accumulates mean and covariance of the neighbourhood in the reference's order and
// arithmetic (core/covariance.hpp:121-135), solves the 3x3 symmetric eigenproblem in registers and
// writes the eigenvector of the smallest eigenvalue, oriented towards the view point when one is set.
//
// kNN / kNN-in-radius: the k best (d2, position) pairs live in shared memory ([slot][thread], no bank
// conflicts), ascending (d2, original index) — the order KNNSearchResultAdaptor produces
// (core/kd_tree.hpp:77-99) whenever the neighbour distances are distinct; on exact ties the reference's
// order is its kd-tree traversal order, ours is lowest index first. Covariance: bit-exact in that case.
// Radius: two sweeps (mean, then covariance) in grid order; the reference sums in ascending distance,
// so this mode agrees to fp32 rounding, not bit for bit.
#include "cb_internal.hpp"
#include "grid_sweep.cuh"
#include "normals_out.cuh"
#include <algorithm>
#include <cmath>

using namespace cb;

namespace {

constexpr int kBlock = 128;
constexpr int kMaxK = 128;  // k-best lists in shared memory: 8 B x k x 128 threads (dynamic above 48 KB)

template <int K>
__global__ void __launch_bounds__(kBlock) normals_knn_kernel(const GridView g, int k, float max_d2, const NormalOut o) {
  extern __shared__ __align__(16) unsigned char knn_smem[];
  float(*sd)[kBlock] = reinterpret_cast<float(*)[kBlock]>(knn_smem);
  uint32_t(*sp)[kBlock] = reinterpret_cast<uint32_t(*)[kBlock]>(knn_smem + sizeof(float) * K * kBlock);
  const int t = threadIdx.x;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t qi = blockIdx.x * blockDim.x + t; qi < g.n; qi += stride) {
    const float4 s = __ldg(g.pts + qi);
    const int oi = __float_as_int(s.w);
    int count = 0;
    float worst = max_d2;  // strict admission bound until the list is full, then the k-th distance
    auto orig = [&](uint32_t pos) { return __float_as_int(__ldg(&g.pts[pos].w)); };
    auto bound = [&]() { return worst; };
    auto scan = [&](uint32_t b, uint32_t e) {
      for (uint32_t j = b; j < e; ++j) {
        const float4 p = __ldg(g.pts + j);
        const float r = rule::contract_d2(s.x, s.y, s.z, p.x, p.y, p.z);
        if (!(r < max_d2)) continue;
        const int pi = __float_as_int(p.w);
        if (count == k) {
          if (r > worst) continue;
          if (r == worst && pi > orig(sp[k - 1][t])) continue;
        }
        int pos = (count < k) ? count : k - 1;
        while (pos > 0) {
          const float pd = sd[pos - 1][t];
          if (pd > r || (pd == r && orig(sp[pos - 1][t]) > pi)) {
            sd[pos][t] = pd;
            sp[pos][t] = sp[pos - 1][t];
            --pos;
          } else {
            break;
          }
        }
        sd[pos][t] = r;
        sp[pos][t] = j;
        if (count < k) ++count;
        if (count == k) worst = sd[k - 1][t];
      }
    };
    grid_sweep(
        g, s.x, s.y, s.z, bound, scan,
        [&]() {
          count = 0;
          worst = max_d2;
        },
        (uint32_t)k);
    float cv[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const bool valid = count >= 3;  // setMinValidSampleSize(points_.rows()), normal_estimation.hpp:27
    if (valid) {
      float mx = 0.f, my = 0.f, mz = 0.f;
      for (int j = 0; j < count; j++) {
        const float4 p = __ldg(g.pts + sp[j][t]);
        mx = __fadd_rn(mx, p.x);
        my = __fadd_rn(my, p.y);
        mz = __fadd_rn(mz, p.z);
      }
      const float inv = __fdiv_rn(1.0f, (float)count);
      mx = __fmul_rn(inv, mx);
      my = __fmul_rn(inv, my);
      mz = __fmul_rn(inv, mz);
      for (int j = 0; j < count; j++) {
        const float4 p = __ldg(g.pts + sp[j][t]);
        const float dx = __fsub_rn(p.x, mx), dy = __fsub_rn(p.y, my), dz = __fsub_rn(p.z, mz);
        cv[0] = __fadd_rn(cv[0], __fmul_rn(dx, dx));
        cv[1] = __fadd_rn(cv[1], __fmul_rn(dx, dy));
        cv[2] = __fadd_rn(cv[2], __fmul_rn(dx, dz));
        cv[3] = __fadd_rn(cv[3], __fmul_rn(dy, dy));
        cv[4] = __fadd_rn(cv[4], __fmul_rn(dy, dz));
        cv[5] = __fadd_rn(cv[5], __fmul_rn(dz, dz));
      }
      const float invm1 = __fdiv_rn(1.0f, (float)(count - 1));
#pragma unroll
      for (int c = 0; c < 6; c++) cv[c] = __fmul_rn(invm1, cv[c]);
    }
    finish_point(o, qi, oi, s.x, s.y, s.z, valid, cv);
  }
}

__global__ void __launch_bounds__(kBlock) normals_radius_kernel(const GridView g, float r2, const NormalOut o) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t qi = blockIdx.x * blockDim.x + threadIdx.x; qi < g.n; qi += stride) {
    const float4 s = __ldg(g.pts + qi);
    const int oi = __float_as_int(s.w);
    auto bound = [&]() { return r2; };
    auto dist2 = [&](const float4& p) { return rule::contract_d2(s.x, s.y, s.z, p.x, p.y, p.z); };
    int count = 0;
    float mx = 0.f, my = 0.f, mz = 0.f;
    grid_sweep(g, s.x, s.y, s.z, bound, [&](uint32_t b, uint32_t e) {
      for (uint32_t j = b; j < e; ++j) {
        const float4 p = __ldg(g.pts + j);
        if (dist2(p) < r2) {
          mx += p.x;
          my += p.y;
          mz += p.z;
          ++count;
        }
      }
    }, [&]() {
      count = 0;
      mx = my = mz = 0.f;
    }, 0u);
    float cv[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const bool valid = count >= 3;
    if (valid) {
      const float inv = __fdiv_rn(1.0f, (float)count);
      mx = __fmul_rn(inv, mx);
      my = __fmul_rn(inv, my);
      mz = __fmul_rn(inv, mz);
      grid_sweep(g, s.x, s.y, s.z, bound, [&](uint32_t b, uint32_t e) {
        for (uint32_t j = b; j < e; ++j) {
          const float4 p = __ldg(g.pts + j);
          if (dist2(p) < r2) {
            const float dx = __fsub_rn(p.x, mx), dy = __fsub_rn(p.y, my), dz = __fsub_rn(p.z, mz);
            cv[0] = __fadd_rn(cv[0], __fmul_rn(dx, dx));
            cv[1] = __fadd_rn(cv[1], __fmul_rn(dx, dy));
            cv[2] = __fadd_rn(cv[2], __fmul_rn(dx, dz));
            cv[3] = __fadd_rn(cv[3], __fmul_rn(dy, dy));
            cv[4] = __fadd_rn(cv[4], __fmul_rn(dy, dz));
            cv[5] = __fadd_rn(cv[5], __fmul_rn(dz, dz));
          }
        }
      }, [&]() {
#pragma unroll
        for (int c = 0; c < 6; c++) cv[c] = 0.f;
      }, 0u);
      const float invm1 = __fdiv_rn(1.0f, (float)(count - 1));
#pragma unroll
      for (int c = 0; c < 6; c++) cv[c] = __fmul_rn(invm1, cv[c]);
    }
    finish_point(o, qi, oi, s.x, s.y, s.z, valid, cv);
  }
}

}  // namespace

extern "C" int cb_cloud_estimate_normals(cb_context* ctx, cb_cloud* cloud, int k, float radius2,
                                         const float* view_point3, int use_current_as_ref, float* normals,
                                         float* curvature, float* cov6, float* gpu_ms) {
  CB_CHECK(ctx && cloud, CB_ERR_INVALID, "null argument");
  CB_CHECK(cloud->ctx == ctx, CB_ERR_INVALID, "cloud belongs to another context");
  CB_CHECK(k >= 0 && k <= kMaxK, CB_ERR_UNSUPPORTED, "k must be in [0, 128] (0 = radius neighbourhood)");
  CB_CHECK(k > 0 || radius2 > 0.f, CB_ERR_INVALID, "need k > 0 and/or radius2 > 0");
  CB_CUDA(cudaSetDevice(ctx->device));
  if (gpu_ms) *gpu_ms = 0.f;
  const size_t n = cloud->n;
  if (n == 0) return CB_OK;
  CB_TRY(ensure_index(cloud));
  const bool use_ref = use_current_as_ref && cloud->d_nrm;  // like PointCloud: only when normals exist
  if (!cloud->d_raw_nrm) CB_TRY(cloud->mem.alloc(&cloud->d_raw_nrm, 3 * n));
  if (!cloud->d_nrm) CB_TRY(cloud->mem.alloc(&cloud->d_nrm, n));
  DeviceScope scope(ctx);
  float* d_curv = nullptr;
  float* d_cov = nullptr;
  if (curvature) CB_TRY(scope.alloc(&d_curv, n));
  if (cov6) CB_TRY(scope.alloc(&d_cov, 6 * n));
  NormalOut o;
  o.raw_nrm = cloud->d_raw_nrm;
  o.nrm = cloud->d_nrm;
  o.curvature = d_curv;
  o.cov6 = d_cov;
  set_orientation(o, view_point3, use_ref);
  const float max_d2 = radius2 > 0.f ? radius2 : 3.402823466e38f;
  const GridView g = grid_view(cloud);
  const int blocks = (int)std::max<size_t>(1, std::min<size_t>((size_t)ctx->sm_count * 8, (n + kBlock - 1) / kBlock));
  ScopedEvents ev;
  if (gpu_ms) {
    CB_TRY(ev.create());
    CB_CUDA(cudaEventRecord(ev.e0, ctx->stream));
  }
  if (k == 0)
    normals_radius_kernel<<<blocks, kBlock, 0, ctx->stream>>>(g, max_d2, o);
  else if (k <= 8)
    normals_knn_kernel<8><<<blocks, kBlock, 8 * kBlock * 8, ctx->stream>>>(g, k, max_d2, o);
  else if (k <= 16)
    normals_knn_kernel<16><<<blocks, kBlock, 16 * kBlock * 8, ctx->stream>>>(g, k, max_d2, o);
  else if (k <= 32)
    normals_knn_kernel<32><<<blocks, kBlock, 32 * kBlock * 8, ctx->stream>>>(g, k, max_d2, o);
  else if (k <= 64) {
    // (per call, not once per process: function attributes belong to the device the context is on)
    CB_CUDA(cudaFuncSetAttribute(normals_knn_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * kBlock * 8));
    normals_knn_kernel<64><<<blocks, kBlock, 64 * kBlock * 8, ctx->stream>>>(g, k, max_d2, o);
  } else {
    CB_CUDA(cudaFuncSetAttribute(normals_knn_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * kBlock * 8));
    normals_knn_kernel<128><<<blocks, kBlock, 128 * kBlock * 8, ctx->stream>>>(g, k, max_d2, o);
  }
  ctx->launches += 1;
  if (gpu_ms) CB_CUDA(cudaEventRecord(ev.e1, ctx->stream));
  CB_CUDA(cudaGetLastError());
  if (normals)
    CB_CUDA(cudaMemcpyAsync(normals, cloud->d_raw_nrm, 3 * n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  if (curvature)
    CB_CUDA(cudaMemcpyAsync(curvature, d_curv, n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  if (cov6) CB_CUDA(cudaMemcpyAsync(cov6, d_cov, 6 * n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  if (gpu_ms) CB_CUDA(cudaEventElapsedTime(gpu_ms, ev.e0, ev.e1));
  return CB_OK;
}
