// Projective correspondence search of rigid ICP (CorrespondenceSearchProjective, correspondence_search/
// correspondence_search_projective.hpp:156-209) under the contract of DESIGN §4.21 (product code, sm_90a).
//
// build_projective_map builds the index map over the destination cloud ONCE per attach (cb_icp_set_projection and the
// warp-field objects' set_projection, warp_field_common.cuh): the z-buffer of pointsToIndexMap
// (depth_images.cu, index_map_keys: smallest camera z, lowest original index on ties, non-finite points skipped), then
// one pass turns each pixel's winner into its position in the destination's cell-sorted arrays (4 B per pixel, -1
// empty), so that the passes gather from the same arrays as the kd-tree paths. Per source point the search is O(1):
// q = T s (rule::transform_point), the pixel q lands in (project_pixel, projection.hpp), one map read and the contract
// distance to that one destination point, kept iff d2 < max_d2.
//   launch_projective_search  per-query result: the host-driven loop's passes (icp_pass_kernel without search) and
//                             the list path of icp_engine.cu read it; the warp-field ICPs run it on their warped
//                             points with the identity (warp_search, DESIGN §4.22)
//   icp_projective_kernel     the device-resident loop's pass (icp_loop.cu)
#include "icp_kernels.cuh"
#include "icp_object.hpp"
#include "launch.cuh"
#include <cmath>

namespace cb {

namespace {

constexpr int kThreads = 256;

// inv[original index] = sorted position
__global__ void inverse_order_kernel(const float4* __restrict__ pts, uint32_t n, uint32_t* __restrict__ inv) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x)
    inv[__float_as_uint(__ldg(&pts[p].w))] = p;
}

// map[k] = sorted position of pixel k's winner, -1 where the pixel is empty
__global__ void index_map_positions_kernel(const unsigned long long* __restrict__ keys, size_t npix,
                                           const uint32_t* __restrict__ inv, int* __restrict__ map) {
  for (size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x; k < npix; k += (size_t)gridDim.x * blockDim.x) {
    const unsigned long long key = keys[k];
    map[k] = key == ~0ull ? -1 : (int)inv[(uint32_t)key];
  }
}

__global__ void __launch_bounds__(kThreads) projective_search_kernel(const Projection prj, const int* __restrict__ map,
                                                                     const float4* __restrict__ src_pts,
                                                                     uint32_t n_src, const float4* __restrict__ dst_pts,
                                                                     const Rigid T, float max_d2, int* nn_pos,
                                                                     float* nn_d2, int* out_idx, float* out_d2) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_src; i += gridDim.x * blockDim.x) {
    const float4 s = __ldg(src_pts + i);
    float qx, qy, qz;
    rule::transform_point(T, s.x, s.y, s.z, qx, qy, qz);
    int pos = -1;
    float d2 = max_d2;
    uint32_t px, py;
    float cz;
    if (project_pixel(prj, qx, qy, qz, px, py, cz)) {
      const int m = __ldg(map + (size_t)py * prj.w + px);
      if (m >= 0) {
        const float4 p = __ldg(dst_pts + m);
        const float v = rule::contract_d2(qx, qy, qz, p.x, p.y, p.z);
        if (v < max_d2) {
          pos = m;
          d2 = v;
        }
      }
    }
    if (nn_pos) nn_pos[i] = pos;
    if (nn_d2) nn_d2[i] = d2;
    const uint32_t oi = __float_as_uint(s.w);
    if (out_idx) out_idx[oi] = pos >= 0 ? __float_as_int(__ldg(&dst_pts[pos].w)) : -1;
    if (out_d2) out_d2[oi] = d2;
  }
}

bool all_finite(const float* v, int n) {
  for (int i = 0; i < n; i++)
    if (!std::isfinite(v[i])) return false;
  return true;
}

}  // namespace

int launch_projective_search(cb_context* ctx, const ProjectiveMap& pm, const float4* src_pts, uint32_t n_src,
                             const float4* dst_pts, const Rigid& T, float max_d2, int* nn_pos, float* nn_d2,
                             int* out_idx, float* out_d2) {
  if (n_src == 0) return CB_OK;
  return launch(ctx, projective_search_kernel, grid_for(ctx, n_src, kThreads), kThreads, 0, pm.prj,
                (const int*)pm.d_map, src_pts, n_src, dst_pts, T, max_d2, nn_pos, nn_d2, out_idx, out_d2);
}

int build_projective_map(cb_context* ctx, DeviceScope& owner, const cb_cloud* dst, const float* K9, size_t w, size_t h,
                         const float* E12, ProjectiveMap* out) {
  CB_CHECK(all_finite(K9, 9), CB_ERR_INVALID, "intrinsics are not finite");
  CB_CHECK(!E12 || all_finite(E12, 12), CB_ERR_INVALID, "extrinsics are not finite");
  CB_CHECK(w < (1ull << 32) && h < (1ull << 32) && (unsigned __int128)w * h < ((unsigned __int128)1 << 32),
           CB_ERR_INVALID, "images of >= 2^32 pixels are not supported");
  ProjectiveMap pm;
  pm.on = true;
  pm.prj = make_projection(K9, E12, (uint32_t)w, (uint32_t)h);
  const size_t npix = w * h, nd = dst->n;
  CB_TRY(owner.alloc(&pm.d_map, npix));
  auto build = [&]() -> int {
    if (npix == 0) return CB_OK;  // no pixel: no correspondences
    DeviceScope scope(ctx);
    unsigned long long* keys = nullptr;
    uint32_t* inv = nullptr;
    CB_TRY(scope.alloc(&keys, npix));
    CB_TRY(scope.alloc(&inv, nd));
    CB_TRY(index_map_keys(ctx, dst->d_raw, nd, pm.prj, keys));
    if (nd)
      CB_TRY(launch(ctx, inverse_order_kernel, grid_for(ctx, nd, kThreads), kThreads, 0, (const float4*)dst->d_pts,
                    (uint32_t)nd, inv));
    CB_TRY(launch(ctx, index_map_positions_kernel, grid_for(ctx, npix, kThreads), kThreads, 0,
                  (const unsigned long long*)keys, npix, (const uint32_t*)inv, pm.d_map));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    return CB_OK;
  };
  const int rc = build();
  if (rc != CB_OK) {
    owner.free(pm.d_map);
    return rc;
  }
  *out = pm;
  return CB_OK;
}

}  // namespace cb

using namespace cb;

int cb_icp_set_projection(cb_icp* icp, const float* K9, size_t w, size_t h, const float* E12) {
  CB_CHECK(icp, CB_ERR_INVALID, "null argument");
  cb_context* ctx = icp->ctx;
  CB_CHECK(ctx->world == 1, CB_ERR_UNSUPPORTED, "projective correspondence search with several ranks");
  CB_CUDA(cudaSetDevice(ctx->device));
  // the new map is built beside the attached one, which stays in force when the build fails
  ProjectiveMap next;  // K9 == NULL: detached, the kd-tree paths
  if (K9) CB_TRY(build_projective_map(ctx, icp->mem, icp->dst, K9, w, h, E12, &next));
  // the object's search changes: nothing it found before describes the new one
  CB_TRY(icp->mem.free(icp->proj.d_map));
  icp->proj = next;
  icp->nn_valid = false;
  icp->nn_stored = false;
  icp->warm_ok = false;
  icp->engine_last = false;
  icp->loop_last = false;
  return CB_OK;
}
