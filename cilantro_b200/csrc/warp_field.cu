// Non-rigid ICP with a dense rigid warp field on the device (product code, sm_90a). DESIGN §4.13.
//
// Replaces CombinedMetricDenseWarpFieldICP<RigidTransform<float, 3>> (registration/
// icp_warp_field_combined_metric_dense.hpp) and the 3-D rigid overload of estimateDenseWarpFieldCombinedMetric
// (registration/warp_field_estimation.hpp:368-715). The reference builds an Eigen sparse Jacobian At per
// Gauss-Newton step, forms At At^T and runs Eigen's Jacobi-preconditioned CG on one thread. Here the normal
// equations are never formed as a sparse matrix; their structure is used directly:
//   * a data row touches one point: the data terms give a dense 6x6 block B_i and a 6-vector g_i per point;
//   * a regularisation row touches two points with opposite diagonal entries: arc e = (lo, hi) adds
//     c_e = h'^2 (6 values) to both diagonal blocks and -c_e to the two couplings,
// so (At At^T p)_i = B_i p_i + sum_{arcs e at i} c_e (p_i - p_other(e)).
// Per Gauss-Newton step: warp_assemble_kernel (one thread per point: B_i, g_i, the preconditioner and the c_e of the
// arcs it is the lower end of), then warp_cg_kernel, one cooperative launch that runs the whole CG loop with grid
// syncs between the matvec, the dot products and the vector updates, and adds the solution to the unknowns. The host
// reads one small record per step (the exact max of |delta_i|^2, the CG iteration count). Per ICP iteration the
// search is the grid 1-NN of the ICP pass kernel on the warped points, and warp_compose_kernel turns the unknowns into
// transforms, applies them and warps the points for the next search.
//
// Arithmetic: vectors, blocks and the assembly are fp32 like the reference's scalar type, every operation rounded on
// its own (no FMA contraction), so that the serial oracle (oracle/warp_field_oracle.cpp) can restate it. Dot products
// and norms are fp64, summed in a fixed order (per thread, then a warp tree, then the blocks in index order), and no
// float atomics are used: results are bit-identical from run to run. sin, cos and exp are taken in double and rounded
// to float (the reference's float std::sin / std::exp are within one ulp of that).
#include "warp_field_common.cuh"
#include <cstring>

// The dense field: one block of unknowns per source point (m = n), nothing beyond the shared core.
struct cb_warp_icp : WarpCore {
  using WarpCore::WarpCore;
};

namespace {

struct AssembleArgs {
  uint32_t n;
  const float* dst_raw;
  const float* dst_nrm;
  const float4* warped;
  const int* corr_dst;        // slot k: dst index or < 0 (no correspondence)
  const uint32_t* corr_off;   // CSR of the slots per point, or nullptr: slot i belongs to point i
  const float* xs;
  const uint32_t* inc_off;
  const uint32_t* inc_arc;
  const uint32_t* inc_other;
  const float* arc_d2;
  float* arc_c;
  float* B;
  float* b;
  float* inv;
  float w_pt_sqrt, w_pl_sqrt, reg_sqrt, reg_coeff, huber;
  bool use_pt, use_pl;
  WarpStats* stats;
};

__global__ void __launch_bounds__(kBlock) warp_assemble_kernel(const AssembleArgs a) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  float x[6];
#pragma unroll
  for (int u = 0; u < 6; u++) x[u] = a.xs[6 * (size_t)i + u];
  float B[21], g[6];
#pragma unroll
  for (int u = 0; u < 21; u++) B[u] = 0.f;
#pragma unroll
  for (int u = 0; u < 6; u++) g[u] = 0.f;

  const uint32_t k0 = a.corr_off ? a.corr_off[i] : i, k1 = a.corr_off ? a.corr_off[i + 1] : i + 1;
  unsigned int found = 0;
  if (a.use_pt || a.use_pl) {
    for (uint32_t k = k0; k < k1; k++) {
      const int j = a.corr_dst[k];
      if (j < 0) continue;
      ++found;
      const float4 s4 = a.warped[i];
      const float s[3] = {s4.x, s4.y, s4.z};
      // sqrt(w) * sqrt(UnityWeightEvaluator = 1) on both the Jacobian and the residual (:496-600)
      add_data_rows(x, s, a.dst_raw, a.dst_nrm, j, a.use_pt, a.use_pl, a.w_pt_sqrt, a.w_pt_sqrt, a.w_pl_sqrt,
                    a.w_pl_sqrt, B, g);
    }
  }
  if (found) atomicAdd(&a.stats->num_corr, found);  // integer: order-free

  float diag[6];
#pragma unroll
  for (int u = 0; u < 6; u++) diag[u] = B[upper_index(u, u)];
  // regularisation (:603-673)
  for (uint32_t k = a.inc_off[i]; k < a.inc_off[i + 1]; k++) {
    const uint32_t e = a.inc_arc[k], o = a.inc_other[k];
    const bool lo = i < o;
    float xo[6], c[6];
#pragma unroll
    for (int u = 0; u < 6; u++) xo[u] = a.xs[6 * (size_t)o + u];
    add_arc(x, xo, lo, arc_weight(a.reg_sqrt, a.reg_coeff, a.arc_d2[e]), a.huber, diag, g, c);
    if (lo)
#pragma unroll
      for (int u = 0; u < 6; u++) a.arc_c[6 * (size_t)e + u] = c[u];
  }
#pragma unroll
  for (int u = 0; u < 21; u++) a.B[21 * (size_t)i + u] = B[u];
#pragma unroll
  for (int u = 0; u < 6; u++) {
    a.b[6 * (size_t)i + u] = g[u];
    a.inv[6 * (size_t)i + u] = diag[u] != 0.f ? __fdiv_rn(1.f, diag[u]) : 1.f;  // DiagonalPreconditioner
  }
}

struct CgArgs {
  CgVecs v;
  const float* B;
  const uint32_t* inc_off;
  const uint32_t* inc_arc;
  const uint32_t* inc_other;
  const float* arc_c;
};

// One Gauss-Newton step's CG (pcg) with (At At^T p)_i = B_i p_i + sum_{arcs e at i} c_e (p_i - p_other(e)).
__global__ void __launch_bounds__(kBlock) warp_cg_kernel(const CgArgs a) {
  cg::grid_group grid = cg::this_grid();
  pcg(a.v, grid, [=]() {
    const uint32_t stride = gridDim.x * blockDim.x;
    double v = 0.0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.v.n; i += stride) {
      float p[6], q[6];
      load6(a.v.p, i, p);
      const float* Bi = a.B + 21 * (size_t)i;
#pragma unroll
      for (int r = 0; r < 6; r++) {
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < 6; c++) s = fa(s, fm(__ldg(Bi + (r <= c ? upper_index(r, c) : upper_index(c, r))), p[c]));
        q[r] = s;
      }
      for (uint32_t k = __ldg(a.inc_off + i), k1 = __ldg(a.inc_off + i + 1); k < k1; k++) {
        const uint32_t e = __ldg(a.inc_arc + k), o = __ldg(a.inc_other + k);
        float po[6];
        load6(a.v.p, o, po);
#pragma unroll
        for (int u = 0; u < 6; u++) q[u] = fa(q[u], fm(__ldg(a.arc_c + 6 * (size_t)e + u), fs(p[u], po[u])));
      }
#pragma unroll
      for (int u = 0; u < 6; u++) v += (double)p[u] * (double)q[u];
      store6(a.v.q, i, q);
    }
    return v;
  });
}

// One estimateDenseWarpFieldCombinedMetric call (gauss_newton) with the dense assembly and CG.
int dense_gauss_newton(cb_warp_icp* w, const cb_warp_params* p, const int* corr_dst, const uint32_t* corr_off,
                       bool no_corr, GnCounts* gn) {
  cb_context* ctx = w->ctx;
  AssembleArgs aa{};
  aa.n = w->n;
  aa.dst_raw = w->dst->d_raw;
  aa.dst_nrm = w->dst->d_raw_nrm;
  aa.warped = w->d_warped;
  aa.corr_dst = corr_dst;
  aa.corr_off = corr_off;
  aa.xs = w->d_xs;
  aa.inc_off = w->d_inc_off;
  aa.inc_arc = w->d_inc_arc;
  aa.inc_other = w->d_inc_other;
  aa.arc_d2 = w->d_arc_d2;
  aa.arc_c = w->d_arc_c;
  aa.B = w->d_B;
  aa.b = w->d_b;
  aa.inv = w->d_inv;
  aa.w_pt_sqrt = sqrtf(p->w_pt);
  aa.w_pl_sqrt = sqrtf(p->w_pl);
  aa.reg_sqrt = sqrtf(p->stiffness);
  aa.reg_coeff = p->reg_coeff;
  aa.huber = p->huber;
  aa.use_pt = p->w_pt > 0.f;
  aa.use_pl = p->w_pl > 0.f;
  aa.stats = w->d_stats;
  CgArgs ca{};
  ca.B = w->d_B;
  ca.inc_off = w->d_inc_off;
  ca.inc_arc = w->d_inc_arc;
  ca.inc_other = w->d_inc_other;
  ca.arc_c = w->d_arc_c;
  auto assemble = [&]() -> int {
    warp_assemble_kernel<<<(unsigned)(((size_t)w->n + kBlock - 1) / kBlock), kBlock, 0, ctx->stream>>>(aa);
    ctx->launches += 1;
    CB_CUDA(cudaGetLastError());
    return CB_OK;
  };
  return gauss_newton(w, p, no_corr, assemble, (const void*)warp_cg_kernel, ca, gn, nullptr);
}

}  // namespace

extern "C" {

void cb_warp_default_params(cb_warp_params* p) {
  if (!p) return;
  std::memset(p, 0, sizeof(*p));
  p->w_pt = 0.f;   // icp_warp_field_combined_metric_dense.hpp (constructor)
  p->w_pl = 1.f;
  p->stiffness = 1.f;
  p->huber = 1e-4f;
  p->max_gn_iter = 10;
  p->gn_tol = 1e-5f;
  p->max_cg_iter = 1000;
  p->cg_tol = 1e-5f;
  p->max_iter = 15;                  // icp_base.hpp:24
  p->tol = 1e-5f;                    // icp_base.hpp:25
  p->max_d2 = (float)(0.01 * 0.01);  // correspondence_search_kd_tree.hpp:49
  p->reg_coeff = -0.5f;              // RBFKernelWeightEvaluator() (common_pair_evaluators.hpp:51)
  p->search_dir = CB_SECOND_TO_FIRST;
  p->inlier_fraction = 1.0;
}

int cb_warp_icp_create(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src, const uint64_t* reg_offsets,
                       const int64_t* reg_index, const float* reg_value, size_t n_reg, cb_warp_icp** out) {
  CB_CHECK(ctx && dst && src && out, CB_ERR_INVALID, "null argument");
  CB_TRY(check_warp_clouds(ctx, dst, src));
  const uint32_t n = (uint32_t)src->n;
  std::vector<uint32_t> lo, hi;
  std::vector<float> d2;
  CB_TRY(build_arcs(n, reg_offsets, reg_index, reg_value, n_reg, lo, hi, d2));
  return create_object(ctx, dst, src, n, (uint32_t)lo.size(), out, [&](cb_warp_icp* w) {
    CB_TRY(alloc_core(w, (const void*)warp_cg_kernel, n));
    return upload_arc_incidence(w, lo, hi, d2);
  });
}

void cb_warp_icp_destroy(cb_warp_icp* w) { destroy_object(w); }

int cb_warp_icp_estimate(cb_warp_icp* w, const cb_warp_params* p, const float* T_init, float* T_out,
                         cb_warp_result* res) {
  CB_TRY(check_params(w, p));
  CB_CHECK(res && (w->n == 0 || T_out), CB_ERR_INVALID, "null argument");
  cb_context* ctx = w->ctx;
  const uint64_t launches0 = ctx->launches;
  ScopedEvents ev_s, ev_v;
  CB_TRY(ev_s.create());
  CB_TRY(ev_v.create());
  std::memset(res, 0, sizeof(*res));
  double ms_search = 0, ms_solve = 0;
  CB_TRY(warp_points(w, w->d_T, T_init));  // transform_ = transform_init_ (icp_base.hpp:72)
  float last_delta = INFINITY;
  int it = 0;
  uint32_t num_corr = 0;
  GnCounts gn;
  while (it < p->max_iter) {
    CB_CUDA(cudaEventRecord(ev_s.e0, ctx->stream));
    CB_TRY(warp_search(w, p->max_d2));  // updateCorrespondences
    CB_CUDA(cudaEventRecord(ev_s.e1, ctx->stream));
    CB_CUDA(cudaEventRecord(ev_v.e0, ctx->stream));
    CB_TRY(dense_gauss_newton(w, p, w->d_nn, nullptr, false, &gn));
    float ld2 = 0.f;
    CB_TRY(apply_update(w, true, true, &ld2, &num_corr));  // preApply + last_delta_norm_
    CB_CUDA(cudaEventRecord(ev_v.e1, ctx->stream));
    CB_CUDA(cudaEventSynchronize(ev_v.e1));
    float a = 0.f, b = 0.f;
    CB_CUDA(cudaEventElapsedTime(&a, ev_s.e0, ev_s.e1));
    CB_CUDA(cudaEventElapsedTime(&b, ev_v.e0, ev_v.e1));
    ms_search += a;
    ms_solve += b;
    last_delta = sqrtf(ld2);
    it++;
    if (last_delta < p->tol) break;
  }
  w->have_corr = it > 0;
  if (w->n) CB_CUDA(cudaMemcpyAsync(T_out, w->d_T, 12 * (size_t)w->n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  res->iterations = it;
  res->last_delta = last_delta;
  res->converged = it > 0 && last_delta < p->tol;
  res->num_corr = num_corr;
  res->gn_steps = gn.steps;
  res->cg_iterations = gn.cg_total;
  res->gpu_ms_search = ms_search;
  res->gpu_ms_solve = ms_solve;
  res->kernel_launches = ctx->launches - launches0;
  return CB_OK;
}

int cb_warp_icp_solve(cb_warp_icp* w, const cb_warp_params* p, const float* T_src, const uint64_t* corr_first,
                      const uint64_t* corr_second, const float* corr_value, size_t n_corr, float* T_out, float* x_out,
                      cb_warp_solve_result* res) {
  (void)corr_value;  // UnityWeightEvaluator ignores the value
  CB_TRY(check_params(w, p));
  CB_CHECK(res && (w->n == 0 || T_out) && (n_corr == 0 || (corr_first && corr_second)), CB_ERR_INVALID,
           "null argument");
  CB_CHECK(n_corr < 0x7fffffffull, CB_ERR_UNSUPPORTED, "too many correspondences");
  cb_context* ctx = w->ctx;
  const uint64_t launches0 = ctx->launches;
  std::memset(res, 0, sizeof(*res));
  CorrSlots cs(ctx);
  CB_TRY(upload_corr_slots(w, corr_first, corr_second, n_corr, &cs));
  CB_TRY(warp_points(w, w->d_T, T_src));
  GnCounts gn;
  CB_TRY(dense_gauss_newton(w, p, cs.d_slot, cs.d_off, n_corr == 0, &gn));
  float ld2 = 0.f;
  CB_TRY(apply_update(w, false, false, &ld2, nullptr));
  if (w->n) CB_CUDA(cudaMemcpyAsync(T_out, w->d_T, 12 * (size_t)w->n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  if (w->n && x_out)
    CB_CUDA(cudaMemcpyAsync(x_out, w->d_xs, 6 * (size_t)w->n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  res->converged = gn.converged;
  res->gn_steps = gn.steps;
  res->cg_iterations = gn.cg_total;
  res->cg_iterations_last = gn.cg_last;
  res->cg_error = gn.cg_err;
  res->kernel_launches = ctx->launches - launches0;
  return CB_OK;
}

int cb_warp_icp_residuals(cb_warp_icp* w, const cb_warp_params* p, const float* T, float* out) {
  CB_TRY(check_params(w, p));
  CB_CHECK(w->n == 0 || (T && out), CB_ERR_INVALID, "null argument");
  if (w->n == 0) return CB_OK;
  CB_TRY(warp_points(w, w->d_T, T));
  return warp_residuals(w, p, out);
}

int cb_warp_icp_correspondences(cb_warp_icp* w, uint64_t* index_first, uint64_t* index_second, float* value,
                                size_t* count) {
  return warp_correspondences(w, index_first, index_second, value, count);
}

}  // extern "C"
