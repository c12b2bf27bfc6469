// Fused ICP iteration kernels (product code, sm_90a).
//
// One launch per ICP iteration does, for every source point s_i:
//   q_i = T s_i                               transformFeatures + transformPoints
//                                             (common_transformable_feature_adaptors.hpp:28-34,
//                                              core/space_transformations.hpp:203-216)
//   (j, d2) = radius-bounded 1-NN of q_i      findNNCorrespondencesUnidirectional
//                                             (correspondence_search_kd_tree_utilities.hpp:26-33)
//   keep iff found and d2 < max_d2            (:29)
//   accumulate the estimator's moments        Kabsch: transform_estimation.hpp:25-34
//                                             Gauss-Newton: :298-343 (combined), :669-715 (symmetric)
// and reduces them warp -> block -> grid (last-block pattern) in double precision. The serial
// stream compaction of the reference (:45-50) disappears: the accumulation is order-free and the
// correspondence list is only materialised when a caller asks for it.
#include "icp_accumulate.cuh"
#include "icp_kernels.cuh"
#include "reduce.cuh"
#include "warp_search.cuh"
#include <algorithm>

namespace cb {

namespace {

constexpr int kBlock = kReduceBlock;

// cp.async.bulk.prefetch.L2: one instruction asks the memory system to pull `bytes` (multiple of 16,
// 16-byte aligned address) from HBM into L2 without occupying registers or a scoreboard slot.
__device__ __forceinline__ void bulk_prefetch_l2(const void* p, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}

constexpr int kIcpMinBlocks = 5;  // resident blocks per SM the pass kernel's register budget is set for

template <int MODE, bool SEARCH>
__global__ void __launch_bounds__(kBlock, kIcpMinBlocks) icp_pass_kernel(const IcpArgs a, const bool has_pt, const bool has_pl) {
  constexpr int NV = (MODE == kModeP2P || MODE == kModeP2PCentered) ? kP2PValues : (MODE == kModeCombined ? kCombinedValues : 1);
  double acc[NV];
#pragma unroll
  for (int i = 0; i < NV; i++) acc[i] = 0.0;

  // ONE query per thread: the moment accumulators are dead during the search, so the search runs at
  // a low register count. Blocks own 256 consecutive queries of the cell-sorted source cloud, i.e. a
  // compact spatial neighbourhood (L1 reuse of the reference cells).
  __shared__ WarpSearchSmem wsm[SEARCH ? kBlock / 32 : 1];
  __shared__ AsyncReduceSmem<NV> rsm;
  if constexpr (MODE != kModeKnn) {
    if (a.rs.ex.trace && blockIdx.x == 0 && threadIdx.x == 0) a.rs.ex.trace[0] = global_timer_ns();  // kernel start
    async_reduce_init(rsm);
  }
  if (SEARCH && threadIdx.x == 0 && a.dst.n > 0) {
    // Software prefetch of the reference arrays into L2, a fixed number of blocks ahead of the
    // consumer front. Both clouds are cell-sorted x-major in (nearly) the same frame, so block b of
    // the query cloud reads the reference arrays around the fraction b / gridDim.x; the bulk
    // prefetch turns the first-touch DRAM latency of the dependent cell-table -> point loads into an
    // L2 hit. A hint only: DRAM traffic and results are unchanged.
    const uint32_t nb = gridDim.x, D = a.prefetch_blocks;
    const uint32_t n_dst = a.dst.n;
    const uint32_t ncells = (uint32_t)a.dst.nx * (uint32_t)a.dst.ny * (uint32_t)a.dst.nz;
    auto prefetch_slice = [&](uint32_t blk) {
      const uint32_t lo = (uint32_t)(((unsigned long long)blk * n_dst) / nb);
      const uint32_t hi = (uint32_t)(((unsigned long long)(blk + 1) * n_dst) / nb);
      if (hi > lo) {
        bulk_prefetch_l2(a.dst.pts + lo, (hi - lo) * 16u);
        if (MODE == kModeCombined && a.dst.nrm) bulk_prefetch_l2(a.dst.nrm + lo, (hi - lo) * 16u);
      }
      const uint32_t clo = (uint32_t)(((unsigned long long)blk * ncells) / nb) & ~3u;
      const uint32_t chi = min(ncells, ((uint32_t)(((unsigned long long)(blk + 1) * ncells) / nb) + 3u) & ~3u);
      if (chi > clo + 3u) bulk_prefetch_l2(a.dst.cell_start + clo, ((chi - clo) & ~3u) * 4u);
    };
    if (blockIdx.x + D < nb) prefetch_slice(blockIdx.x + D);
    if (blockIdx.x < D) prefetch_slice(blockIdx.x);  // the first D blocks have nobody ahead of them
  }
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool active = i < a.n_src;
  const float4 s = active ? __ldg(a.src_pts + i) : make_float4(0.f, 0.f, 0.f, 0.f);
  float qx, qy, qz;
  rule::transform_point(a.T, s.x, s.y, s.z, qx, qy, qz);
  int pos = -1;
  float cd2 = 0.f;  // the correspondence's value (squared distance): input of the RBF weight evaluators
  if (SEARCH) {
    // every lane of the warp takes part in the pooled search (inactive tail lanes contribute no work)
    const int warm = (a.warm_pos && active) ? a.warm_pos[i] : -1;
    const Best best = warp_grid_nearest(a.dst, wsm[threadIdx.x >> 5], active, qx, qy, qz, a.max_d2, warm);
    if (active) {
      pos = (best.idx >= 0 && best.d2 < a.max_d2) ? best.pos : -1;
      cd2 = best.d2;
      if (a.nn_pos) a.nn_pos[i] = pos;
      if (a.nn_d2) a.nn_d2[i] = best.d2;
      if (MODE == kModeKnn) {
        const int oi = __float_as_int(s.w);
        if (a.out_idx) a.out_idx[oi] = (pos >= 0) ? best.idx : -1;
        if (a.out_d2) a.out_d2[oi] = (pos >= 0) ? best.d2 : a.max_d2;
      }
    }
  } else if (active) {
    pos = a.nn_pos[i];
    if (MODE == kModeCombined && (a.wk_pt | a.wk_pl) && a.nn_d2) cd2 = a.nn_d2[i];
  }
  if constexpr (MODE != kModeKnn) {
    if (pos >= 0) {
      const float4 dp = __ldg(a.dst.pts + pos);
      accumulate_pair<MODE>(
          acc, a, has_pt, has_pl, dp, qx, qy, qz, a.src_nrm != nullptr, [&] { return __ldg(a.dst.nrm + pos); },
          [&] { return __ldg(a.src_nrm + i); }, cd2);
    }
  }
  if constexpr (MODE != kModeKnn) grid_reduce_async<NV>(acc, a.rs, rsm);
}

__global__ void __launch_bounds__(kBlock) residual_kernel(const GridView dst, const float4* __restrict__ src_pts,
                                                          const float4* __restrict__ src_nrm, uint32_t n_src,
                                                          const Rigid T, int metric, float w_pt, float w_pl,
                                                          float* __restrict__ out) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_src; i += stride) {
    const float4 s = __ldg(src_pts + i);
    const int oi = __float_as_int(s.w);
    float qx, qy, qz;
    rule::transform_point(T, s.x, s.y, s.z, qx, qy, qz);
    const Best best = grid_nearest(dst, qx, qy, qz, 3.402823466e+38f);
    float res = __int_as_float(0x7fc00000);  // NaN when dst is empty (icp_*_metric.hpp:221-224)
    if (best.idx >= 0) {
      const float4 dp = __ldg(dst.pts + best.pos);
      const float e0 = __fsub_rn(dp.x, qx), e1 = __fsub_rn(dp.y, qy), e2 = __fsub_rn(dp.z, qz);
      const float sq = sum3(__fmul_rn(e0, e0), __fmul_rn(e1, e1), __fmul_rn(e2, e2));
      if (metric == CB_ICP_POINT_TO_POINT) {
        res = sq;
      } else {
        const float4 np = __ldg(dst.nrm + best.pos);
        float n0 = np.x, n1 = np.y, n2 = np.z;
        if (src_nrm) {  // the reference adds the UN-rotated source normal here (:236)
          const float4 sn = __ldg(src_nrm + i);
          n0 = __fadd_rn(n0, sn.x);
          n1 = __fadd_rn(n1, sn.y);
          n2 = __fadd_rn(n2, sn.z);
        }
        const float pd = sum3(__fmul_rn(n0, e0), __fmul_rn(n1, e1), __fmul_rn(n2, e2));
        res = __fadd_rn(__fmul_rn(w_pt, sq), __fmul_rn(__fmul_rn(w_pl, pd), pd));
      }
    }
    out[oi] = res;
  }
}

__global__ void transform_points_kernel(const Rigid T, const float* __restrict__ in, size_t n, float* __restrict__ out) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float qx, qy, qz;
    rule::transform_point(T, in[3 * i], in[3 * i + 1], in[3 * i + 2], qx, qy, qz);
    out[3 * i] = qx;
    out[3 * i + 1] = qy;
    out[3 * i + 2] = qz;
  }
}

__global__ void translate_matches_kernel(const int* __restrict__ nn_pos, const float* __restrict__ nn_d2,
                                         const float4* __restrict__ src_pts, const float4* __restrict__ dst_pts,
                                         uint32_t n_src, int* __restrict__ out_first, float* __restrict__ out_val) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n_src; p += gridDim.x * blockDim.x) {
    const int oi = __float_as_int(__ldg(&src_pts[p].w));
    const int pos = nn_pos[p];
    out_first[oi] = pos >= 0 ? __float_as_int(__ldg(&dst_pts[pos].w)) : -1;
    if (out_val) out_val[oi] = nn_d2 ? nn_d2[p] : 0.f;
  }
}

}  // namespace

int launch_translate_matches(cb_context* ctx, const int* nn_pos, const float* nn_d2, const float4* src_pts,
                             const float4* dst_pts, uint32_t n_src, int* out_first, float* out_val) {
  if (n_src == 0) return CB_OK;
  const int blocks = (int)std::max<uint32_t>(1, std::min<uint32_t>((uint32_t)ctx->sm_count * 8, (n_src + 255) / 256));
  translate_matches_kernel<<<blocks, 256, 0, ctx->stream>>>(nn_pos, nn_d2, src_pts, dst_pts, n_src, out_first, out_val);
  ctx->launches += 1;
  CB_CUDA(cudaGetLastError());
  return CB_OK;
}

int icp_grid_blocks(const cb_context* ctx) {
  // persistent-style launch: a whole number of waves of resident CTAs
  static int per_sm = -1;
  if (per_sm < 0) {
    int v = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, icp_pass_kernel<kModeCombined, true>, kBlock, 0) !=
            cudaSuccess ||
        v < 1)
      v = 2;
    per_sm = v;
  }
  return ctx->sm_count * per_sm;
}

int launch_icp_pass(cb_context* ctx, const IcpArgs& a, int mode, bool search, bool has_pt, bool has_pl) {
  if (a.n_src == 0 && mode == kModeKnn) return CB_OK;
  // one query per thread; the hardware block scheduler balances the (variable-cost) searches
  const int blocks = std::max(1, (int)((a.n_src + kBlock - 1) / kBlock));
  IcpArgs args = a;
  CB_TRY(get_reduce_scratch(ctx, blocks, kMaxValues, &args.rs));
  // reduction passes carry the fused NVLink all-reduce + host mailbox epilogue when the context has it
  ctx->pass_armed = (mode != kModeKnn) && arm_exchange(ctx, &args.rs.ex);
  args.prefetch_blocks = (uint32_t)(2 * ctx->sm_count * kIcpMinBlocks);  // ~2 waves of resident blocks
  if (mode == kModeKnn) {
    icp_pass_kernel<kModeKnn, true><<<blocks, kBlock, 0, ctx->stream>>>(args, false, false);
  } else if (mode == kModeP2P) {
    if (search)
      icp_pass_kernel<kModeP2P, true><<<blocks, kBlock, 0, ctx->stream>>>(args, false, false);
    else
      icp_pass_kernel<kModeP2P, false><<<blocks, kBlock, 0, ctx->stream>>>(args, false, false);
  } else if (mode == kModeP2PCentered) {  // Kabsch moments about the pivots a.dm / a.sm (the ICP loop; always a search pass)
    icp_pass_kernel<kModeP2PCentered, true><<<blocks, kBlock, 0, ctx->stream>>>(args, false, false);
  } else {
    if (search)
      icp_pass_kernel<kModeCombined, true><<<blocks, kBlock, 0, ctx->stream>>>(args, has_pt, has_pl);
    else
      icp_pass_kernel<kModeCombined, false><<<blocks, kBlock, 0, ctx->stream>>>(args, has_pt, has_pl);
  }
  ctx->launches += 1;
  CB_CUDA(cudaGetLastError());
  return CB_OK;
}

int launch_residuals(cb_context* ctx, const GridView& dst, const float4* src_pts, const float4* src_nrm,
                     uint32_t n_src, const Rigid& T, int metric, float w_pt, float w_pl, float* d_out) {
  if (n_src == 0) return CB_OK;
  int blocks = std::max(1, std::min(icp_grid_blocks(ctx), (int)((n_src + kBlock - 1) / kBlock)));
  residual_kernel<<<blocks, kBlock, 0, ctx->stream>>>(dst, src_pts, src_nrm, n_src, T, metric, w_pt, w_pl, d_out);
  ctx->launches += 1;
  CB_CUDA(cudaGetLastError());
  return CB_OK;
}

int launch_transform_points(cb_context* ctx, const Rigid& T, const float* d_in, size_t n, float* d_out) {
  if (n == 0) return CB_OK;
  int blocks = (int)std::max<size_t>(1, std::min<size_t>((size_t)ctx->sm_count * 8, (n + 255) / 256));
  transform_points_kernel<<<blocks, 256, 0, ctx->stream>>>(T, d_in, n, d_out);
  ctx->launches += 1;
  CB_CUDA(cudaGetLastError());
  return CB_OK;
}

}  // namespace cb
