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

struct cb_warp_icp {
  explicit cb_warp_icp(cb_context* c) : ctx(c), mem(c) {}
  cb_context* ctx = nullptr;
  cb::DeviceScope mem;  // every buffer below (device and pinned host)
  const cb_cloud* dst = nullptr;
  const cb_cloud* src = nullptr;
  uint32_t n = 0;        // source points
  uint32_t n_arcs = 0;   // regularisation arcs (self-arcs dropped)
  // arcs (lo < hi) and their incidence, sorted stably by point: entries inc_off[i] .. inc_off[i+1]-1 of point i
  uint32_t* d_arc_lo = nullptr;
  uint32_t* d_arc_hi = nullptr;
  float* d_arc_d2 = nullptr;
  float* d_arc_c = nullptr;  // [n_arcs][6] c_e of the current step
  uint32_t* d_inc_off = nullptr;
  uint32_t* d_inc_arc = nullptr;
  uint32_t* d_inc_other = nullptr;
  // per point
  float* d_T = nullptr;       // [n][12] current transforms
  float4* d_warped = nullptr; // T_i s_i, .w = index bits (the search's query layout)
  float* d_xs = nullptr;      // [n][6] unknowns of the running estimator call
  float* d_B = nullptr;       // [n][21] data block, upper triangle row-major
  float* d_b = nullptr;       // [n][6] right-hand side At b
  float* d_inv = nullptr;     // [n][6] Jacobi preconditioner
  float* d_vec = nullptr;     // [5][n][6] CG vectors x, r, p, z, q
  int* d_nn = nullptr;        // [n] last search: dst index or -1
  float* d_nn_d2 = nullptr;
  double* d_part = nullptr;   // CG reduction partials [5][grid]
  WarpStats* d_stats = nullptr;
  WarpStats* h_stats = nullptr;  // pinned
  int cg_grid = 0;
  bool have_corr = false;
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

int check_params(const cb_warp_icp* w, const cb_warp_params* p) {
  CB_CHECK(w && p, CB_ERR_INVALID, "null argument");
  return check_warp_params(w->ctx, w->dst, p);
}

// One estimateDenseWarpFieldCombinedMetric call on the current warped points and correspondence slots (the unknowns
// start at zero, :460-461). Returns the estimator's flag through *converged and accumulates the step and CG counts.
// corr_known: the host knows whether the list is empty (has_corr); else the first step's assembly counts it.
int gauss_newton(cb_warp_icp* w, const cb_warp_params* p, const int* corr_dst, const uint32_t* corr_off, bool corr_known,
                 bool has_corr, int* converged, uint64_t* steps, uint64_t* cg_total, uint64_t* cg_last, float* cg_err) {
  cb_context* ctx = w->ctx;
  WarpStats* hs = (WarpStats*)w->h_stats;
  const size_t n = w->n;
  *converged = 0;
  CB_CUDA(cudaMemsetAsync(w->d_xs, 0, 6 * std::max<size_t>(n, 1) * sizeof(float), ctx->stream));
  const bool use_pt = p->w_pt > 0.f, use_pl = p->w_pl > 0.f;
  if ((!use_pt && !use_pl) || (corr_known && !has_corr) || n == 0) return CB_OK;  // :398-408
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
  aa.use_pt = use_pt;
  aa.use_pl = use_pl;
  aa.stats = (WarpStats*)w->d_stats;
  CgArgs ca{};
  ca.v.n = w->n;
  ca.v.b = w->d_b;
  ca.v.inv = w->d_inv;
  ca.v.x = w->d_vec;
  ca.v.r = w->d_vec + 6 * n;
  ca.v.p = w->d_vec + 12 * n;
  ca.v.z = w->d_vec + 18 * n;
  ca.v.q = w->d_vec + 24 * n;
  ca.v.xs = w->d_xs;
  ca.v.part = w->d_part;
  ca.v.max_iter = (unsigned int)std::min<uint64_t>(p->max_cg_iter, 0xffffffffu);
  ca.v.tol = (double)p->cg_tol;
  ca.v.stats = (WarpStats*)w->d_stats;
  ca.B = w->d_B;
  ca.inc_off = w->d_inc_off;
  ca.inc_arc = w->d_inc_arc;
  ca.inc_other = w->d_inc_other;
  ca.arc_c = w->d_arc_c;
  const float tol2 = p->gn_tol * p->gn_tol;
  for (uint64_t step = 0; step < p->max_gn_iter; step++) {
    CB_CUDA(cudaMemsetAsync(w->d_stats, 0, sizeof(WarpStats), ctx->stream));
    warp_assemble_kernel<<<(unsigned)((n + kBlock - 1) / kBlock), kBlock, 0, ctx->stream>>>(aa);
    CB_CUDA(cudaGetLastError());
    void* args[] = {&ca};
    CB_CUDA(cudaLaunchCooperativeKernel((const void*)warp_cg_kernel, dim3(w->cg_grid), dim3(kBlock), args, 0, ctx->stream));
    ctx->launches += 2;
    CB_CUDA(cudaMemcpyAsync(hs, w->d_stats, sizeof(WarpStats), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    // no correspondence: b = 0, so the step left xs at zero; the reference returns before any step
    if (step == 0 && hs->num_corr == 0) return CB_OK;
    ++*steps;
    *cg_total += hs->cg_iters;
    *cg_last = hs->cg_iters;
    *cg_err = hs->cg_err;
    float mx;
    std::memcpy(&mx, &hs->max_delta_bits, sizeof(float));
    if (mx < tol2) {
      *converged = 1;
      break;
    }
  }
  return CB_OK;
}

int apply_update(cb_warp_icp* w, bool compose, bool warp_next, float* last_delta_sq, uint32_t* num_corr) {
  cb_context* ctx = w->ctx;
  WarpStats* hs = (WarpStats*)w->h_stats;
  CB_CUDA(cudaMemsetAsync(w->d_stats, 0, sizeof(WarpStats), ctx->stream));
  if (w->n) {
    warp_compose_kernel<<<grid_for(ctx, w->n), kBlock, 0, ctx->stream>>>(
        w->n, w->src->d_raw, w->d_xs, w->d_T, compose, warp_next ? w->d_warped : nullptr, warp_next ? w->d_nn : nullptr,
        (WarpStats*)w->d_stats);
    ctx->launches += 1;
    CB_CUDA(cudaGetLastError());
  }
  CB_CUDA(cudaMemcpyAsync(hs, w->d_stats, sizeof(WarpStats), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  std::memcpy(last_delta_sq, &hs->last_delta_bits, sizeof(float));
  *num_corr = hs->num_corr;
  return CB_OK;
}

int warp_points(cb_warp_icp* w, const float* T_host) {
  cb_context* ctx = w->ctx;
  if (w->n == 0) return CB_OK;
  if (T_host)
    CB_CUDA(cudaMemcpyAsync(w->d_T, T_host, 12 * (size_t)w->n * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  warp_points_kernel<<<grid_for(ctx, w->n), kBlock, 0, ctx->stream>>>(w->n, w->src->d_raw, w->d_T, T_host == nullptr,
                                                                      w->d_warped);
  ctx->launches += 1;
  CB_CUDA(cudaGetLastError());
  return CB_OK;
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

// Device buffers of a new warp-field ICP object: arcs (lo, hi, d2) uploaded and their incidence sorted by point.
static int warp_init(cb_warp_icp* w, const std::vector<uint32_t>& lo, const std::vector<uint32_t>& hi,
                     const std::vector<float>& d2) {
  cb_context* ctx = w->ctx;
  const uint32_t n = w->n;
  const size_t nn = std::max<size_t>(n, 1), m = std::max<size_t>(w->n_arcs, 1);
  CB_TRY(w->mem.alloc(&w->d_arc_lo, m));
  CB_TRY(w->mem.alloc(&w->d_arc_hi, m));
  CB_TRY(w->mem.alloc(&w->d_arc_d2, m));
  CB_TRY(w->mem.alloc(&w->d_arc_c, 6 * m));
  CB_TRY(w->mem.alloc(&w->d_inc_off, nn + 1));
  CB_TRY(w->mem.alloc(&w->d_inc_arc, 2 * m));
  CB_TRY(w->mem.alloc(&w->d_inc_other, 2 * m));
  CB_TRY(w->mem.alloc(&w->d_T, 12 * nn));
  CB_TRY(w->mem.alloc(&w->d_warped, nn));
  CB_TRY(w->mem.alloc(&w->d_xs, 6 * nn));
  CB_TRY(w->mem.alloc(&w->d_B, 21 * nn));
  CB_TRY(w->mem.alloc(&w->d_b, 6 * nn));
  CB_TRY(w->mem.alloc(&w->d_inv, 6 * nn));
  CB_TRY(w->mem.alloc(&w->d_vec, 30 * nn));
  CB_TRY(w->mem.alloc(&w->d_nn, nn));
  CB_TRY(w->mem.alloc(&w->d_nn_d2, nn));
  CB_TRY(w->mem.alloc(&w->d_stats, 1));
  CB_TRY(w->mem.alloc_host(&w->h_stats, 1));
  // cooperative grid: every block resident (occupancy API), no more blocks than points need
  int per_sm = 0;
  CB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, warp_cg_kernel, kBlock, 0));
  CB_CHECK(per_sm >= 1, CB_ERR_CUDA, "the CG kernel cannot be resident");
  w->cg_grid = (int)std::max<size_t>(1, std::min<size_t>((size_t)ctx->sm_count * per_sm, (nn + kBlock - 1) / kBlock));
  CB_TRY(w->mem.alloc(&w->d_part, 5 * (size_t)w->cg_grid));
  return upload_arc_incidence(ctx, n, lo, hi, d2, w->d_arc_lo, w->d_arc_hi, w->d_arc_d2, w->d_inc_off, w->d_inc_arc,
                              w->d_inc_other);
}

int cb_warp_icp_create(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src, const uint64_t* reg_offsets,
                       const int64_t* reg_index, const float* reg_value, size_t n_reg, cb_warp_icp** out) {
  CB_CHECK(ctx && dst && src && out, CB_ERR_INVALID, "null argument");
  CB_TRY(check_warp_clouds(ctx, dst, src));
  const uint32_t n = (uint32_t)src->n;
  std::vector<uint32_t> lo, hi;
  std::vector<float> d2;
  CB_TRY(build_arcs(n, reg_offsets, reg_index, reg_value, n_reg, lo, hi, d2));
  CB_CUDA(cudaSetDevice(ctx->device));
  CB_TRY(ensure_index(const_cast<cb_cloud*>(dst)));
  cb_warp_icp* w = new cb_warp_icp(ctx);
  w->dst = dst;
  w->src = src;
  w->n = n;
  w->n_arcs = (uint32_t)lo.size();
  const int rc = warp_init(w, lo, hi, d2);
  if (rc != CB_OK) {
    delete w;
    return rc;
  }
  *out = w;
  return CB_OK;
}

void cb_warp_icp_destroy(cb_warp_icp* w) {
  if (!w) return;
  cudaSetDevice(w->ctx->device);
  cudaStreamSynchronize(w->ctx->stream);
  delete w;
}

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
  CB_TRY(warp_points(w, T_init));  // transform_ = transform_init_ (icp_base.hpp:72)
  float last_delta = INFINITY;
  int it = 0;
  uint32_t num_corr = 0;
  while (it < p->max_iter) {
    CB_CUDA(cudaEventRecord(ev_s.e0, ctx->stream));
    CB_TRY(warp_search(ctx, w->dst, w->d_warped, w->n, p->max_d2, w->d_nn, w->d_nn_d2));  // updateCorrespondences
    CB_CUDA(cudaEventRecord(ev_s.e1, ctx->stream));
    CB_CUDA(cudaEventRecord(ev_v.e0, ctx->stream));
    int conv = 0;
    uint64_t cg_last = 0;
    float cg_err = 0.f;
    CB_TRY(gauss_newton(w, p, w->d_nn, nullptr, false, false, &conv, &res->gn_steps, &res->cg_iterations, &cg_last,
                        &cg_err));
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
  std::vector<uint32_t> off;
  std::vector<int> slot;
  CB_TRY(corr_slots(w->dst->n, w->n, corr_first, corr_second, n_corr, off, slot));
  DeviceScope scope(ctx);
  uint32_t* d_off = nullptr;
  int* d_slot = nullptr;
  CB_TRY(scope.alloc(&d_off, off.size()));
  CB_TRY(scope.alloc(&d_slot, slot.size()));
  CB_CUDA(cudaMemcpyAsync(d_off, off.data(), off.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
  CB_CUDA(cudaMemcpyAsync(d_slot, slot.data(), slot.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
  CB_TRY(warp_points(w, T_src));
  int conv = 0;
  uint32_t nc = 0;
  CB_TRY(gauss_newton(w, p, d_slot, d_off, true, n_corr > 0, &conv, &res->gn_steps, &res->cg_iterations,
                      &res->cg_iterations_last, &res->cg_error));
  float ld2 = 0.f;
  CB_TRY(apply_update(w, false, false, &ld2, &nc));
  if (w->n) CB_CUDA(cudaMemcpyAsync(T_out, w->d_T, 12 * (size_t)w->n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  if (w->n && x_out)
    CB_CUDA(cudaMemcpyAsync(x_out, w->d_xs, 6 * (size_t)w->n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  res->converged = conv;
  res->kernel_launches = ctx->launches - launches0;
  return CB_OK;
}

int cb_warp_icp_residuals(cb_warp_icp* w, const cb_warp_params* p, const float* T, float* out) {
  CB_TRY(check_params(w, p));
  CB_CHECK(w->n == 0 || (T && out), CB_ERR_INVALID, "null argument");
  if (w->n == 0) return CB_OK;
  CB_TRY(warp_points(w, T));
  return warp_residuals(w->ctx, w->dst, w->d_warped, w->n, p, out);
}

int cb_warp_icp_correspondences(cb_warp_icp* w, uint64_t* index_first, uint64_t* index_second, float* value,
                                size_t* count) {
  CB_CHECK(w && count, CB_ERR_INVALID, "null argument");
  CB_CHECK(w->have_corr, CB_ERR_INVALID, "no estimate() has run");
  return warp_correspondences(w->ctx, w->n, w->d_nn, w->d_nn_d2, index_first, index_second, value, count);
}

}  // extern "C"
