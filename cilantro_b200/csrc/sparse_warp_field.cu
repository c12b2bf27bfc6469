// Non-rigid ICP with a sparse, control-node rigid warp field on the device (product code, sm_90a). DESIGN §4.14.
//
// Replaces CombinedMetricSparseWarpFieldICP<RigidTransform<float, 3>> (registration/
// icp_warp_field_combined_metric_sparse.hpp), resampleTransforms (registration/warp_field_utilities.hpp:14-48) and the
// 3-D rigid overload of estimateSparseWarpFieldCombinedMetric (registration/warp_field_estimation.hpp:1388-1846).
// The unknowns are 6 per control node; source point i blends the unknowns of its control list with the weights
// w_ik = exp(ctrl_coeff d2_ik) / W_i. Its data rows are those of the dense estimator evaluated at the blend, with the
// entry of node n_ik scaled by w_ik, so with W_i = [w_i1 I6 ... w_iK I6] the normal equations are
//   (At At^T p)_j = sum_i (W_i^T B_i W_i p)_j + sum_{arcs e at j} c_e (p_j - p_other(e)),
// B_i the point's 6x6 data block (already scaled by (corr_weight_sqrt / W_i)^2). They are never formed as a matrix:
//   * sparse_assemble_kernel (one thread per point): the blended linearisation point, B_i and g_i;
//   * sparse_node_kernel (one thread per node): b_j = sum_i w_ij g_i + arc terms, the Jacobi diagonal
//     sum_i (sum of w_ij over the point's list)^2 diag(B_i) + sum_e c_e, and the arcs' c_e;
//   * sparse_cg_kernel: one cooperative launch per Gauss-Newton step running the whole CG; its matvec is
//     P_i = sum_k w_ik p_{n_ik}, y_i = B_i P_i (per point), a grid sync, then q_j = sum w_ij y_i + arcs (per node).
// The node->(point, slot) incidence is built once, by the stable radix sort keyed by node, so every gather runs in a
// fixed order. Per ICP iteration: the search of the dense path on the warped points (grid 1-NN, or projective with a
// projection attached), the Gauss-Newton steps,
// warp_compose_kernel over the nodes (preApply with projection, the last_delta max) and sparse_resample_kernel (node
// transforms -> per-point transforms -> warped points for the next search).
//
// Arithmetic as in warp_field.cu (warp_field_common.cuh): fp32 without FMA contraction where the serial oracle
// (oracle/sparse_warp_field_oracle.cpp) restates the order, fp64 dot products in a fixed order, no float atomics.
#include "warp_field_common.cuh"
#include <cstring>

// The sparse field: the core's blocks are the m control nodes; the control lists and the per-point buffers here.
struct cb_sparse_warp_icp : WarpCore {
  using WarpCore::WarpCore;
  uint32_t nnz = 0;  // control-list entries
  // control lists: per point entries ctrl_off[i] .. ctrl_off[i+1]-1, in the given order (resampling, W_i) and sorted
  // stably by node (the estimator: sidx[k] = node, sperm[k] = the given entry it came from)
  uint32_t* d_ctrl_off = nullptr;
  uint32_t* d_ctrl_idx = nullptr;
  float* d_ctrl_d2 = nullptr;
  uint32_t* d_sidx = nullptr;
  uint32_t* d_sperm = nullptr;
  float* d_w = nullptr;    // [nnz] exp(ctrl_coeff d2), given order
  float* d_ws = nullptr;   // [nnz] the same, sorted order
  float* d_W = nullptr;    // [n] total weight (summed in the given order)
  // node -> (point, sorted entry), ascending entry: entries ninc_off[j] .. ninc_off[j+1]-1 of node j
  uint32_t* d_ninc_off = nullptr;
  uint32_t* d_ninc_pt = nullptr;
  uint32_t* d_ninc_slot = nullptr;
  // per point
  float* d_Td = nullptr;  // [n][12] dense warp field
  float* d_g = nullptr;   // [n][6]
  float* d_y = nullptr;   // [n][6] B_i P_i of the running matvec
};

namespace {

// w = RBFKernelWeightEvaluator<float, float, true>(d2) per entry, W_i in list order, and the sorted copy
__global__ void ctrl_weights_kernel(uint32_t n, const uint32_t* __restrict__ off, const float* __restrict__ d2,
                                    const uint32_t* __restrict__ sperm, float coeff, float* __restrict__ w,
                                    float* __restrict__ ws, float* __restrict__ W) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float tot = 0.f;
    for (uint32_t k = off[i]; k < off[i + 1]; k++) {
      const float v = (float)exp((double)fm(coeff, d2[k]));
      w[k] = v;
      tot = fa(tot, v);
    }
    for (uint32_t k = off[i]; k < off[i + 1]; k++) ws[k] = w[sperm[k]];
    W[i] = tot;
  }
}

// resampleTransforms (warp_field_utilities.hpp:14-48): T_i = (rotation(sum_k w_k R_k / W), sum_k w_k t_k / W) over
// the list in the given order, the identity when W = 0; then the warped point T_i s_i and the count of matches in nn.
__global__ void sparse_resample_kernel(uint32_t n, const uint32_t* __restrict__ off, const uint32_t* __restrict__ idx,
                                       const float* __restrict__ w, const float* __restrict__ W,
                                       const float* __restrict__ T, const float* __restrict__ src_raw,
                                       float* __restrict__ Td, float4* __restrict__ warped, const int* __restrict__ nn,
                                       WarpStats* stats) {
  unsigned int found = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (nn && nn[i] >= 0) ++found;
    float L[12];
#pragma unroll
    for (int u = 0; u < 12; u++) L[u] = 0.f;
    for (uint32_t k = off[i]; k < off[i + 1]; k++) {
      const float wk = w[k];
      const float* Tk = T + 12 * (size_t)idx[k];
#pragma unroll
      for (int u = 0; u < 12; u++) L[u] = fa(L[u], fm(wk, Tk[u]));
    }
    const float tot = W[i];
    if (tot == 0.f) {
      sc::t34_identity(L);
    } else {
      const float inv = __fdiv_rn(1.f, tot);
#pragma unroll
      for (int u = 0; u < 12; u++) L[u] = fm(L[u], inv);
      sc::reorthonormalize(L);  // LinearTransform::rotation()
    }
#pragma unroll
    for (int u = 0; u < 12; u++) Td[12 * (size_t)i + u] = L[u];
    const float s[3] = {src_raw[3 * (size_t)i], src_raw[3 * (size_t)i + 1], src_raw[3 * (size_t)i + 2]};
    float q[3];
    sc::apply_point(L, s, q);
    warped[i] = make_float4(q[0], q[1], q[2], __int_as_float((int)i));
  }
  for (int o = 16; o > 0; o >>= 1) found += __shfl_xor_sync(0xffffffffu, found, o);
  if ((threadIdx.x & 31) == 0 && found) atomicAdd(&stats->num_corr, found);
}

struct SparseAssembleArgs {
  uint32_t n;
  const float* dst_raw;
  const float* dst_nrm;
  const float4* warped;
  const int* corr_dst;        // slot k: dst index or < 0
  const uint32_t* corr_off;   // CSR of the slots per point, or nullptr: slot i belongs to point i
  const uint32_t* ctrl_off;
  const uint32_t* sidx;
  const float* ws;
  const float* W;
  const float* xs;            // node unknowns
  float* B;
  float* g;
  float w_pt_sqrt, w_pl_sqrt;
  bool use_pt, use_pl;
  WarpStats* stats;
};

// Data rows of one source point (:1568-1731): linearised at (sum_k w_k x_{n_k}) (1/W) over the sorted list, Jacobian
// scaled by corr_weight_sqrt / W (the node's w_k is applied by the node pass and the matvec), residual by
// corr_weight_sqrt; both zero when W = 0.
__global__ void __launch_bounds__(kBlock) sparse_assemble_kernel(const SparseAssembleArgs a) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  float B[21], g[6];
#pragma unroll
  for (int u = 0; u < 21; u++) B[u] = 0.f;
#pragma unroll
  for (int u = 0; u < 6; u++) g[u] = 0.f;
  const uint32_t k0 = a.corr_off ? a.corr_off[i] : i, k1 = a.corr_off ? a.corr_off[i + 1] : i + 1;
  unsigned int found = 0;
  if (a.use_pt || a.use_pl)
    for (uint32_t k = k0; k < k1; k++) found += a.corr_dst[k] >= 0;
  if (found) {  // only points with a data term need their blend (:1455-1469)
    const float W = a.W[i];
    float x[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float wj_pt = 0.f, wr_pt = 0.f, wj_pl = 0.f, wr_pl = 0.f;
    if (W != 0.f) {
      for (uint32_t k = a.ctrl_off[i]; k < a.ctrl_off[i + 1]; k++) {
        const float wk = a.ws[k];
        const float* xn = a.xs + 6 * (size_t)a.sidx[k];
#pragma unroll
        for (int u = 0; u < 6; u++) x[u] = fa(x[u], fm(wk, xn[u]));
      }
      const float inv = __fdiv_rn(1.f, W);
#pragma unroll
      for (int u = 0; u < 6; u++) x[u] = fm(x[u], inv);
      wr_pt = a.w_pt_sqrt;  // sqrt(w_pt) * sqrt(UnityWeightEvaluator = 1)
      wr_pl = a.w_pl_sqrt;
      wj_pt = __fdiv_rn(wr_pt, W);
      wj_pl = __fdiv_rn(wr_pl, W);
    }
    const float4 s4 = a.warped[i];
    const float s[3] = {s4.x, s4.y, s4.z};
    for (uint32_t k = k0; k < k1; k++) {
      const int j = a.corr_dst[k];
      if (j < 0) continue;
      add_data_rows(x, s, a.dst_raw, a.dst_nrm, j, a.use_pt, a.use_pl, wj_pt, wr_pt, wj_pl, wr_pl, B, g);
    }
    atomicAdd(&a.stats->num_corr, found);  // integer: order-free
  }
#pragma unroll
  for (int u = 0; u < 21; u++) a.B[21 * (size_t)i + u] = B[u];
#pragma unroll
  for (int u = 0; u < 6; u++) a.g[6 * (size_t)i + u] = g[u];
}

struct SparseNodeArgs {
  uint32_t m;
  const uint32_t* ninc_off;
  const uint32_t* ninc_pt;
  const uint32_t* ninc_slot;
  const float* ws;
  const float* B;
  const float* g;
  const float* xs;
  const uint32_t* inc_off;
  const uint32_t* inc_arc;
  const uint32_t* inc_other;
  const float* arc_d2;
  float* arc_c;
  float* b;
  float* inv;
  float reg_sqrt, reg_coeff, huber;
};

// Per node j: b_j = sum_(i,k) w_k g_i + the arcs' share (:1734-1804), the Jacobi diagonal and the c_e of the arcs
// it is the lower end of. A point listing j several times contributes (sum of its w_k)^2 diag(B_i), as At At^T does.
__global__ void __launch_bounds__(kBlock) sparse_node_kernel(const SparseNodeArgs a) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.m) return;
  float b[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, diag[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  uint32_t prev = 0xffffffffu;
  float sw = 0.f;
  for (uint32_t k = a.ninc_off[j], k1 = a.ninc_off[j + 1]; k <= k1; k++) {
    const uint32_t i = k < k1 ? a.ninc_pt[k] : 0xffffffffu;
    if (i != prev && prev != 0xffffffffu) {  // the previous point's group ends
      const float s2 = fm(sw, sw);
#pragma unroll
      for (int u = 0; u < 6; u++) diag[u] = fa(diag[u], fm(s2, a.B[21 * (size_t)prev + upper_index(u, u)]));
      sw = 0.f;
    }
    if (k == k1) break;
    prev = i;
    const float wk = a.ws[a.ninc_slot[k]];
    sw = fa(sw, wk);
#pragma unroll
    for (int u = 0; u < 6; u++) b[u] = fa(b[u], fm(wk, a.g[6 * (size_t)i + u]));
  }
  float x[6];
#pragma unroll
  for (int u = 0; u < 6; u++) x[u] = a.xs[6 * (size_t)j + u];
  for (uint32_t k = a.inc_off[j]; k < a.inc_off[j + 1]; k++) {
    const uint32_t e = a.inc_arc[k], o = a.inc_other[k];
    const bool lo = j < o;
    float xo[6], c[6];
#pragma unroll
    for (int u = 0; u < 6; u++) xo[u] = a.xs[6 * (size_t)o + u];
    add_arc(x, xo, lo, arc_weight(a.reg_sqrt, a.reg_coeff, a.arc_d2[e]), a.huber, diag, b, c);
    if (lo)
#pragma unroll
      for (int u = 0; u < 6; u++) a.arc_c[6 * (size_t)e + u] = c[u];
  }
#pragma unroll
  for (int u = 0; u < 6; u++) {
    a.b[6 * (size_t)j + u] = b[u];
    a.inv[6 * (size_t)j + u] = diag[u] != 0.f ? __fdiv_rn(1.f, diag[u]) : 1.f;  // DiagonalPreconditioner
  }
}

struct SparseCgArgs {
  CgVecs v;                  // over the m nodes
  uint32_t n;                // points
  const uint32_t* ctrl_off;
  const uint32_t* sidx;
  const float* ws;
  const float* B;
  float* y;
  const uint32_t* ninc_off;
  const uint32_t* ninc_pt;
  const uint32_t* ninc_slot;
  const uint32_t* inc_off;
  const uint32_t* inc_arc;
  const uint32_t* inc_other;
  const float* arc_c;
};

// One Gauss-Newton step's CG (pcg) over the node unknowns; the matvec takes one extra grid sync between its point and
// node halves.
__global__ void __launch_bounds__(kBlock) sparse_cg_kernel(const SparseCgArgs a) {
  cg::grid_group grid = cg::this_grid();
  pcg(a.v, grid, [=, &grid]() {
    const uint32_t stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
    for (uint32_t i = t0; i < a.n; i += stride) {  // y_i = B_i (sum_k w_k p_{n_k})
      float P[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (uint32_t k = __ldg(a.ctrl_off + i), k1 = __ldg(a.ctrl_off + i + 1); k < k1; k++) {
        const float wk = __ldg(a.ws + k);
        float pn[6];
        load6(a.v.p, __ldg(a.sidx + k), pn);
#pragma unroll
        for (int u = 0; u < 6; u++) P[u] = fa(P[u], fm(wk, pn[u]));
      }
      const float* Bi = a.B + 21 * (size_t)i;
      float y[6];
#pragma unroll
      for (int r = 0; r < 6; r++) {
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < 6; c++) s = fa(s, fm(__ldg(Bi + (r <= c ? upper_index(r, c) : upper_index(c, r))), P[c]));
        y[r] = s;
      }
      store6(a.y, i, y);
    }
    grid.sync();
    double v = 0.0;
    for (uint32_t j = t0; j < a.v.n; j += stride) {  // q_j = sum w_k y_i + sum_arcs c_e (p_j - p_o)
      float q[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, p[6];
      for (uint32_t k = __ldg(a.ninc_off + j), k1 = __ldg(a.ninc_off + j + 1); k < k1; k++) {
        const float wk = __ldg(a.ws + __ldg(a.ninc_slot + k));
        float y[6];
        load6(a.y, __ldg(a.ninc_pt + k), y);
#pragma unroll
        for (int u = 0; u < 6; u++) q[u] = fa(q[u], fm(wk, y[u]));
      }
      load6(a.v.p, j, p);
      for (uint32_t k = __ldg(a.inc_off + j), k1 = __ldg(a.inc_off + j + 1); k < k1; k++) {
        const uint32_t e = __ldg(a.inc_arc + k), o = __ldg(a.inc_other + k);
        float po[6];
        load6(a.v.p, o, po);
#pragma unroll
        for (int u = 0; u < 6; u++) q[u] = fa(q[u], fm(__ldg(a.arc_c + 6 * (size_t)e + u), fs(p[u], po[u])));
      }
#pragma unroll
      for (int u = 0; u < 6; u++) v += (double)p[u] * (double)q[u];
      store6(a.v.q, j, q);
    }
    return v;
  });
}

// after the sort by node: point and sorted entry per incidence entry, off[j] = first entry of node j (off[m] = total)
__global__ void node_incidence_fill_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                                           uint32_t total, uint32_t m, const uint32_t* __restrict__ slot_pt,
                                           uint32_t* __restrict__ inc_pt, uint32_t* __restrict__ inc_slot,
                                           uint32_t* __restrict__ off) {
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k <= total; k += gridDim.x * blockDim.x) {
    incidence_offsets(keys, k, total, m, off);
    if (k < total) {
      inc_slot[k] = vals[k];
      inc_pt[k] = slot_pt[vals[k]];
    }
  }
}

__global__ void node_keys_kernel(const uint32_t* __restrict__ sidx, uint32_t total, uint64_t* __restrict__ keys,
                                 uint32_t* __restrict__ vals) {
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < total; k += gridDim.x * blockDim.x) {
    keys[k] = sidx[k];
    vals[k] = k;
  }
}

using Obj = cb_sparse_warp_icp;

int check_params(const Obj* w, const cb_sparse_warp_params* p) { return check_params(w, p ? &p->base : nullptr); }

// The control weights of this call's ctrl_coeff.
int weights(Obj* w, const cb_sparse_warp_params* p) {
  if (w->n == 0) return CB_OK;
  return launch(w->ctx, ctrl_weights_kernel, grid_for(w->ctx, w->n, kBlock), kBlock, 0, w->n, w->d_ctrl_off,
                w->d_ctrl_d2, w->d_sperm, p->ctrl_coeff, w->d_w, w->d_ws, w->d_W);
}

// d_T <- T_host (identities when NULL)
int set_nodes(Obj* w, const float* T_host) {
  if (w->m == 0) return CB_OK;
  std::vector<float> I;
  if (!T_host) {
    I.resize(12 * (size_t)w->m);
    for (size_t j = 0; j < w->m; j++) sc::t34_identity(&I[12 * j]);
    T_host = I.data();
  }
  CB_CUDA(cudaMemcpyAsync(w->d_T, T_host, 12 * (size_t)w->m * sizeof(float), cudaMemcpyHostToDevice, w->ctx->stream));
  CB_CUDA(cudaStreamSynchronize(w->ctx->stream));  // I is a pageable host buffer
  return CB_OK;
}

int resample(Obj* w, const int* nn) {
  if (w->n == 0) return CB_OK;
  return launch(w->ctx, sparse_resample_kernel, grid_for(w->ctx, w->n, kBlock), kBlock, 0, w->n, w->d_ctrl_off,
                w->d_ctrl_idx, w->d_w, w->d_W, w->d_T, w->src->d_raw, w->d_Td, w->d_warped, nn, w->d_stats);
}

// One estimateSparseWarpFieldCombinedMetric call (gauss_newton) with the sparse assembly, node pass and CG; the
// control weights of this call must be in place.
int sparse_gauss_newton(Obj* w, const cb_warp_params* p, const int* corr_dst, const uint32_t* corr_off, bool no_corr,
                        GnCounts* gn, StepTimer* timer) {
  cb_context* ctx = w->ctx;
  SparseAssembleArgs aa{};
  aa.n = w->n;
  aa.dst_raw = w->dst->d_raw;
  aa.dst_nrm = w->dst->d_raw_nrm;
  aa.warped = w->d_warped;
  aa.corr_dst = corr_dst;
  aa.corr_off = corr_off;
  aa.ctrl_off = w->d_ctrl_off;
  aa.sidx = w->d_sidx;
  aa.ws = w->d_ws;
  aa.W = w->d_W;
  aa.xs = w->d_xs;
  aa.B = w->d_B;
  aa.g = w->d_g;
  aa.w_pt_sqrt = sqrtf(p->w_pt);
  aa.w_pl_sqrt = sqrtf(p->w_pl);
  aa.use_pt = p->w_pt > 0.f;
  aa.use_pl = p->w_pl > 0.f;
  aa.stats = w->d_stats;
  SparseNodeArgs na{};
  na.m = w->m;
  na.ninc_off = w->d_ninc_off;
  na.ninc_pt = w->d_ninc_pt;
  na.ninc_slot = w->d_ninc_slot;
  na.ws = w->d_ws;
  na.B = w->d_B;
  na.g = w->d_g;
  na.xs = w->d_xs;
  na.inc_off = w->d_inc_off;
  na.inc_arc = w->d_inc_arc;
  na.inc_other = w->d_inc_other;
  na.arc_d2 = w->d_arc_d2;
  na.arc_c = w->d_arc_c;
  na.b = w->d_b;
  na.inv = w->d_inv;
  na.reg_sqrt = sqrtf(p->stiffness);
  na.reg_coeff = p->reg_coeff;
  na.huber = p->huber;
  SparseCgArgs ca{};
  ca.n = w->n;
  ca.ctrl_off = w->d_ctrl_off;
  ca.sidx = w->d_sidx;
  ca.ws = w->d_ws;
  ca.B = w->d_B;
  ca.y = w->d_y;
  ca.ninc_off = w->d_ninc_off;
  ca.ninc_pt = w->d_ninc_pt;
  ca.ninc_slot = w->d_ninc_slot;
  ca.inc_off = w->d_inc_off;
  ca.inc_arc = w->d_inc_arc;
  ca.inc_other = w->d_inc_other;
  ca.arc_c = w->d_arc_c;
  auto assemble = [&]() -> int {
    CB_TRY(launch(ctx, sparse_assemble_kernel, (unsigned)(((size_t)w->n + kBlock - 1) / kBlock), kBlock, 0, aa));
    CB_TRY(launch(ctx, sparse_node_kernel, (unsigned)(((size_t)w->m + kBlock - 1) / kBlock), kBlock, 0, na));
    return CB_OK;
  };
  return gauss_newton(w, p, no_corr, assemble, (const void*)sparse_cg_kernel, ca, gn, timer);
}

int init(Obj* w, const std::vector<uint32_t>& ctrl_off, const std::vector<uint32_t>& ctrl_idx,
         const std::vector<float>& ctrl_d2, const std::vector<uint32_t>& sidx, const std::vector<uint32_t>& sperm,
         const std::vector<uint32_t>& slot_pt, const std::vector<uint32_t>& lo, const std::vector<uint32_t>& hi,
         const std::vector<float>& d2) {
  cb_context* ctx = w->ctx;
  cudaStream_t s = ctx->stream;
  const size_t nn = std::max<size_t>(w->n, 1), mm = std::max<size_t>(w->m, 1), kk = std::max<size_t>(w->nnz, 1);
  CB_TRY(w->mem.alloc(&w->d_ctrl_off, nn + 1));
  CB_TRY(w->mem.alloc(&w->d_ctrl_idx, kk));
  CB_TRY(w->mem.alloc(&w->d_ctrl_d2, kk));
  CB_TRY(w->mem.alloc(&w->d_sidx, kk));
  CB_TRY(w->mem.alloc(&w->d_sperm, kk));
  CB_TRY(w->mem.alloc(&w->d_w, kk));
  CB_TRY(w->mem.alloc(&w->d_ws, kk));
  CB_TRY(w->mem.alloc(&w->d_W, nn));
  CB_TRY(w->mem.alloc(&w->d_ninc_off, mm + 1));
  CB_TRY(w->mem.alloc(&w->d_ninc_pt, kk));
  CB_TRY(w->mem.alloc(&w->d_ninc_slot, kk));
  CB_TRY(w->mem.alloc(&w->d_Td, 12 * nn));
  CB_TRY(w->mem.alloc(&w->d_g, 6 * nn));
  CB_TRY(w->mem.alloc(&w->d_y, 6 * nn));
  // the CG's loops run over the points and over the nodes
  CB_TRY(alloc_core(w, (const void*)sparse_cg_kernel, std::max<size_t>(w->n, w->m)));
  CB_CUDA(cudaMemcpyAsync(w->d_ctrl_off, ctrl_off.data(), ctrl_off.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
  DeviceScope scope(ctx);
  uint32_t* d_slot_pt = nullptr;
  uint64_t *keys = nullptr, *keys_tmp = nullptr;
  uint32_t *vals = nullptr, *vals_tmp = nullptr;
  const uint32_t total = w->nnz;
  CB_TRY(scope.alloc(&d_slot_pt, kk));
  CB_TRY(scope.alloc(&keys, total));
  CB_TRY(scope.alloc(&keys_tmp, total));
  CB_TRY(scope.alloc(&vals, total));
  CB_TRY(scope.alloc(&vals_tmp, total));
  if (total) {
    CB_CUDA(cudaMemcpyAsync(w->d_ctrl_idx, ctrl_idx.data(), total * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CB_CUDA(cudaMemcpyAsync(w->d_ctrl_d2, ctrl_d2.data(), total * sizeof(float), cudaMemcpyHostToDevice, s));
    CB_CUDA(cudaMemcpyAsync(w->d_sidx, sidx.data(), total * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CB_CUDA(cudaMemcpyAsync(w->d_sperm, sperm.data(), total * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CB_CUDA(cudaMemcpyAsync(d_slot_pt, slot_pt.data(), total * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CB_TRY(launch(ctx, node_keys_kernel, grid_for(ctx, total, kBlock), kBlock, 0, w->d_sidx, total, keys, vals));
    int bits = 1;
    while (bits < 32 && (1ull << bits) < (uint64_t)mm) bits++;
    CB_TRY(radix_sort_pairs_u64(ctx, keys, vals, keys_tmp, vals_tmp, total, bits));
  }
  CB_TRY(launch(ctx, node_incidence_fill_kernel, grid_for(ctx, (size_t)total + 1, kBlock), kBlock, 0, keys, vals, total,
                w->m, d_slot_pt, w->d_ninc_pt, w->d_ninc_slot, w->d_ninc_off));
  return upload_arc_incidence(w, lo, hi, d2);  // synchronises the stream
}

int copy_out(Obj* w, float* T_out, float* T_dense_out) {
  cb_context* ctx = w->ctx;
  if (w->m && T_out)
    CB_CUDA(cudaMemcpyAsync(T_out, w->d_T, 12 * (size_t)w->m * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  if (w->n && T_dense_out)
    CB_CUDA(cudaMemcpyAsync(T_dense_out, w->d_Td, 12 * (size_t)w->n * sizeof(float), cudaMemcpyDeviceToHost,
                            ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  return CB_OK;
}

}  // namespace

extern "C" {

void cb_sparse_warp_default_params(cb_sparse_warp_params* p) {
  if (!p) return;
  std::memset(p, 0, sizeof(*p));
  cb_warp_default_params(&p->base);  // icp_warp_field_combined_metric_sparse.hpp (constructor) = the dense defaults
  p->ctrl_coeff = -0.5f;             // RBFKernelWeightEvaluator() (common_pair_evaluators.hpp:51)
}

int cb_sparse_warp_icp_create(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src, const uint64_t* ctrl_offsets,
                              const int64_t* ctrl_index, const float* ctrl_value, size_t n_ctrl_lists, size_t n_ctrl,
                              const uint64_t* reg_offsets, const int64_t* reg_index, const float* reg_value,
                              size_t n_reg, cb_sparse_warp_icp** out) {
  CB_CHECK(ctx && dst && src && out, CB_ERR_INVALID, "null argument");
  CB_TRY(check_warp_clouds(ctx, dst, src));
  CB_CHECK(n_ctrl < 0x7fffffffull, CB_ERR_UNSUPPORTED, "the sparse warp-field ICP supports fewer than 2^31 - 1 nodes");
  const uint32_t n = (uint32_t)src->n, m = (uint32_t)n_ctrl;
  // one control list per source point (the reference would return identities forever and resample to a wrong size)
  CB_CHECK(n_ctrl_lists == n, CB_ERR_INVALID, "one control list per source point expected");
  CB_CHECK(ctrl_offsets, CB_ERR_INVALID, "null control-list offsets");
  CB_CHECK(ctrl_offsets[0] == 0, CB_ERR_INVALID, "control-list offsets must start at 0");
  const uint64_t total = ctrl_offsets[n];
  CB_CHECK(total < 0x7fffffffull, CB_ERR_UNSUPPORTED, "too many control-list entries (2^31 - 1 at most)");
  CB_CHECK(total == 0 || (ctrl_index && ctrl_value), CB_ERR_INVALID, "null control-list index / value");
  std::vector<uint32_t> off((size_t)n + 1), idx(total), sidx(total), sperm(total), slot_pt(total);
  std::vector<float> d2(total);
  for (uint32_t i = 0; i < n; i++) {
    const uint64_t b = ctrl_offsets[i], e = ctrl_offsets[i + 1];
    CB_CHECK(b <= e && e <= total, CB_ERR_INVALID, "control-list offsets must be non-decreasing");
    off[i] = (uint32_t)b;
    for (uint64_t k = b; k < e; k++) {
      CB_CHECK(ctrl_index[k] >= 0 && (uint64_t)ctrl_index[k] < m, CB_ERR_INVALID, "control index outside the nodes");
      idx[k] = (uint32_t)ctrl_index[k];
      d2[k] = ctrl_value[k];
      sperm[k] = (uint32_t)k;
      slot_pt[k] = i;
    }
    // the estimator's sort by index (:1466-1467), stable: duplicates keep their list order
    std::stable_sort(sperm.begin() + b, sperm.begin() + e, [&](uint32_t x, uint32_t y) { return idx[x] < idx[y]; });
    for (uint64_t k = b; k < e; k++) sidx[k] = idx[sperm[k]];
  }
  off[n] = (uint32_t)total;
  std::vector<uint32_t> lo, hi;
  std::vector<float> ad2;
  CB_TRY(build_arcs(m, reg_offsets, reg_index, reg_value, n_reg, lo, hi, ad2));
  return create_object(ctx, dst, src, m, (uint32_t)lo.size(), out, [&](Obj* w) {
    w->nnz = (uint32_t)total;
    return init(w, off, idx, d2, sidx, sperm, slot_pt, lo, hi, ad2);
  });
}

void cb_sparse_warp_icp_destroy(cb_sparse_warp_icp* w) { destroy_object(w); }

int cb_sparse_warp_icp_estimate(cb_sparse_warp_icp* w, const cb_sparse_warp_params* prm, const float* T_init,
                                float* T_out, float* T_dense_out, cb_sparse_warp_result* res) {
  CB_TRY(check_params(w, prm));
  CB_CHECK(res && (w->m == 0 || T_out), CB_ERR_INVALID, "null argument");
  const cb_warp_params* p = &prm->base;
  cb_context* ctx = w->ctx;
  const uint64_t launches0 = ctx->launches;
  ScopedEvents ev_s, ev_r;
  CB_TRY(ev_s.create());
  CB_TRY(ev_r.create());
  std::memset(res, 0, sizeof(*res));
  double ms_search = 0, ms_resample = 0;
  StepTimer times;
  CB_TRY(times.create());
  CB_TRY(weights(w, prm));
  CB_TRY(set_nodes(w, T_init));  // transform_ = transform_init_ (icp_base.hpp:72)
  CB_TRY(resample(w, nullptr));  // initializeComputation (:202-205)
  float last_delta = INFINITY;
  int it = 0;
  uint32_t num_corr = 0;
  GnCounts gn;
  while (it < p->max_iter) {
    CB_CUDA(cudaEventRecord(ev_s.e0, ctx->stream));
    CB_TRY(warp_search(w, p->max_d2));  // updateCorrespondences
    CB_CUDA(cudaEventRecord(ev_s.e1, ctx->stream));
    CB_TRY(sparse_gauss_newton(w, p, w->d_nn, nullptr, false, &gn, &times));
    float ld2 = 0.f;
    CB_TRY(apply_update(w, true, false, &ld2, nullptr));  // preApply over the nodes + last_delta_norm_ (:227, :231-239)
    CB_CUDA(cudaEventRecord(ev_r.e0, ctx->stream));
    CB_CUDA(cudaMemsetAsync(w->d_stats, 0, sizeof(WarpStats), ctx->stream));
    CB_TRY(resample(w, w->d_nn));  // :228-229
    CB_CUDA(cudaEventRecord(ev_r.e1, ctx->stream));
    CB_CUDA(cudaMemcpyAsync(w->h_stats, w->d_stats, sizeof(WarpStats), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaEventSynchronize(ev_r.e1));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    num_corr = w->h_stats->num_corr;
    float a = 0.f, b = 0.f;
    CB_CUDA(cudaEventElapsedTime(&a, ev_s.e0, ev_s.e1));
    CB_CUDA(cudaEventElapsedTime(&b, ev_r.e0, ev_r.e1));
    ms_search += a;
    ms_resample += b;
    last_delta = sqrtf(ld2);
    it++;
    if (last_delta < p->tol) break;
  }
  w->have_corr = it > 0;
  CB_TRY(copy_out(w, T_out, T_dense_out));
  res->iterations = it;
  res->last_delta = last_delta;
  res->converged = it > 0 && last_delta < p->tol;
  res->num_corr = num_corr;
  res->gn_steps = gn.steps;
  res->cg_iterations = gn.cg_total;
  res->gpu_ms_search = ms_search;
  res->gpu_ms_resample = ms_resample;
  res->gpu_ms_assemble = times.assemble;
  res->gpu_ms_cg = times.cg;
  res->kernel_launches = ctx->launches - launches0;
  return CB_OK;
}

int cb_sparse_warp_icp_solve(cb_sparse_warp_icp* w, const cb_sparse_warp_params* prm, const float* T_dense_src,
                             const uint64_t* corr_first, const uint64_t* corr_second, const float* corr_value,
                             size_t n_corr, float* T_out, float* x_out, cb_warp_solve_result* res) {
  (void)corr_value;  // UnityWeightEvaluator ignores the value
  CB_TRY(check_params(w, prm));
  CB_CHECK(res && (w->m == 0 || T_out) && (n_corr == 0 || (corr_first && corr_second)), CB_ERR_INVALID,
           "null argument");
  CB_CHECK(n_corr < 0x7fffffffull, CB_ERR_UNSUPPORTED, "too many correspondences");
  cb_context* ctx = w->ctx;
  const uint64_t launches0 = ctx->launches;
  std::memset(res, 0, sizeof(*res));
  CorrSlots cs(ctx);
  CB_TRY(upload_corr_slots(w, corr_first, corr_second, n_corr, &cs));
  CB_TRY(weights(w, prm));
  CB_TRY(warp_points(w, w->d_Td, T_dense_src));
  GnCounts gn;
  StepTimer times;
  CB_TRY(times.create());
  CB_TRY(sparse_gauss_newton(w, &prm->base, cs.d_slot, cs.d_off, n_corr == 0, &gn, &times));
  float ld2 = 0.f;
  CB_TRY(apply_update(w, false, false, &ld2, nullptr));
  if (w->m && x_out)
    CB_CUDA(cudaMemcpyAsync(x_out, w->d_xs, 6 * (size_t)w->m * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CB_TRY(copy_out(w, T_out, nullptr));
  res->converged = gn.converged;
  res->gn_steps = gn.steps;
  res->cg_iterations = gn.cg_total;
  res->cg_iterations_last = gn.cg_last;
  res->cg_error = gn.cg_err;
  res->kernel_launches = ctx->launches - launches0;
  return CB_OK;
}

int cb_sparse_warp_icp_resample(cb_sparse_warp_icp* w, const cb_sparse_warp_params* prm, const float* T_ctrl,
                                float* T_dense_out) {
  CB_TRY(check_params(w, prm));
  CB_CHECK((w->m == 0 || T_ctrl) && (w->n == 0 || T_dense_out), CB_ERR_INVALID, "null argument");
  CB_TRY(weights(w, prm));
  CB_TRY(set_nodes(w, T_ctrl));
  CB_TRY(resample(w, nullptr));
  return copy_out(w, nullptr, T_dense_out);
}

int cb_sparse_warp_icp_residuals(cb_sparse_warp_icp* w, const cb_sparse_warp_params* prm, const float* T_dense,
                                 float* out) {
  CB_TRY(check_params(w, prm));
  CB_CHECK(w->n == 0 || (T_dense && out), CB_ERR_INVALID, "null argument");
  if (w->n == 0) return CB_OK;
  CB_TRY(warp_points(w, w->d_Td, T_dense));
  return warp_residuals(w, &prm->base, out);
}

int cb_sparse_warp_icp_correspondences(cb_sparse_warp_icp* w, uint64_t* index_first, uint64_t* index_second,
                                       float* value, size_t* count) {
  return warp_correspondences(w, index_first, index_second, value, count);
}

int cb_sparse_warp_icp_set_projection(cb_sparse_warp_icp* w, const float* K9, size_t width, size_t height,
                                      const float* E12) {
  return warp_set_projection(w, K9, width, height, E12);
}

}  // extern "C"
