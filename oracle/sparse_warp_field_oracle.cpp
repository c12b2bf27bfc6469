// ORACLE (test infrastructure, NOT product code): a serial restatement of the 3-D rigid overload of
// estimateSparseWarpFieldCombinedMetric (registration/warp_field_estimation.hpp:1388-1846) and of resampleTransforms
// (registration/warp_field_utilities.hpp:14-48), in the device's fp32 order (sparse_warp_field.cu) or in fp64. The ICP
// loop of CombinedMetricSparseWarpFieldICP and its 1-NN search live in oracle/sparse_warp_field.py.
//
// The reference assembles the sparse At row by row; here, as on the device, each source point i contributes its 6x6
// data block B_i and right-hand side g_i, both already scaled by corr_weight_sqrt / W_i, and node j collects
//   b_j = sum_(i,k: n_ik = j) w_ik g_i,   (A p)_j = sum_(i,k: n_ik = j) w_ik B_i (sum_k' w_ik' p_{n_ik'}) + arcs,
// with the Huber arcs between nodes of the dense restatement (DESIGN §4.14 states why this is At At^T). The Huber rules,
// the rotation terms, the arc list, the correspondence slots and the transform conversion are the dense oracle's.
#include "warp_field_oracle.cpp"

namespace {

template <class S>
struct Ctrl {
  std::vector<uint64_t> off;
  std::vector<uint32_t> idx;   // given order
  std::vector<S> w;            // exp(coeff d2), given order
  std::vector<S> W;            // per point, summed in the given order
  std::vector<uint32_t> sidx;  // sorted stably by node
  std::vector<S> ws;
  std::vector<std::vector<std::pair<uint32_t, uint32_t>>> inc;  // per node: (point, sorted entry), ascending entry
};

template <class S>
Ctrl<S> make_ctrl(size_t n, const uint64_t* off, const int64_t* idx, const float* d2, size_t m, float coeff) {
  Ctrl<S> c;
  c.off.assign(off, off + n + 1);
  const size_t nnz = off[n];
  c.idx.resize(nnz);
  c.w.resize(nnz);
  c.W.assign(n, (S)0);
  c.sidx.resize(nnz);
  c.ws.resize(nnz);
  c.inc.resize(m);
  for (size_t i = 0; i < n; i++) {
    std::vector<uint32_t> perm;
    for (uint64_t k = off[i]; k < off[i + 1]; k++) {
      c.idx[k] = (uint32_t)idx[k];
      c.w[k] = (S)std::exp((double)((S)coeff * (S)d2[k]));
      c.W[i] = c.W[i] + c.w[k];
      perm.push_back((uint32_t)k);
    }
    std::stable_sort(perm.begin(), perm.end(), [&](uint32_t a, uint32_t b) { return c.idx[a] < c.idx[b]; });
    for (size_t t = 0; t < perm.size(); t++) {
      const size_t k = off[i] + t;
      c.sidx[k] = c.idx[perm[t]];
      c.ws[k] = c.w[perm[t]];
      c.inc[c.sidx[k]].push_back({(uint32_t)i, (uint32_t)k});
    }
  }
  return c;
}

template <class S>
struct SparseSystem {
  std::vector<S> B, g;        // per point [n][21] upper, [n][6]
  std::vector<S> b, diag, c;  // per node [m][6], per arc [arcs][6]
};

// the data rows of one correspondence (:1568-1731), Jacobian scaled by wj, residual by wr
template <class S>
void data_rows(const S x[6], const S s[3], const S d[3], const S* nrm, bool pt, S wj_pt, S wr_pt, bool pl, S wj_pl,
               S wr_pl, S* B, S* g) {
  auto add_row = [&](const S J[6], S res) {
    int k = 0;
    for (int r = 0; r < 6; r++) {
      for (int c = r; c < 6; c++, k++) B[k] = B[k] + J[r] * J[c];
      g[r] = g[r] + J[r] * res;
    }
  };
  S M[3][3], Da[3][3], Db[3][3], Dc[3][3];
  rotation_terms<S>(x[0], x[1], x[2], M, Da, Db, Dc);
  S ts[3], das[3], dbs[3], dcs[3];
  for (int r = 0; r < 3; r++) {
    ts[r] = d[r] - (dot3<S>(M[0][r], M[1][r], M[2][r], s[0], s[1], s[2]) + x[3 + r]);
    das[r] = dot3<S>(Da[0][r], Da[1][r], Da[2][r], s[0], s[1], s[2]);
    dbs[r] = dot3<S>(Db[0][r], Db[1][r], Db[2][r], s[0], s[1], s[2]);
    dcs[r] = dot3<S>(Dc[0][r], Dc[1][r], Dc[2][r], s[0], s[1], s[2]);
  }
  if (pt)
    for (int r = 0; r < 3; r++) {
      S J[6] = {das[r] * wj_pt, dbs[r] * wj_pt, dcs[r] * wj_pt, 0, 0, 0};
      J[3 + r] = wj_pt;
      add_row(J, ts[r] * wr_pt);
    }
  if (pl) {
    const S J[6] = {dot3<S>(nrm[0], nrm[1], nrm[2], das[0], das[1], das[2]) * wj_pl,
                    dot3<S>(nrm[0], nrm[1], nrm[2], dbs[0], dbs[1], dbs[2]) * wj_pl,
                    dot3<S>(nrm[0], nrm[1], nrm[2], dcs[0], dcs[1], dcs[2]) * wj_pl,
                    nrm[0] * wj_pl, nrm[1] * wj_pl, nrm[2] * wj_pl};
    add_row(J, dot3<S>(nrm[0], nrm[1], nrm[2], ts[0], ts[1], ts[2]) * wr_pl);
  }
}

template <class S>
void assemble_sparse(const float* dst_p, const float* dst_n, const float* src_p, const CorrCsr& corr, const Ctrl<S>& ctrl,
                     const Arcs& arcs, const Prm& p, bool use_pt, bool use_pl, const std::vector<S>& x,
                     SparseSystem<S>& sys) {
  const size_t n = corr.off.size() - 1, m = ctrl.inc.size();
  sys.B.assign(21 * n, (S)0);
  sys.g.assign(6 * n, (S)0);
  sys.b.assign(6 * m, (S)0);
  sys.diag.assign(6 * m, (S)0);
  sys.c.assign(6 * arcs.lo.size(), (S)0);
  const S w_pt = (S)std::sqrt((S)p.w_pt), w_pl = (S)std::sqrt((S)p.w_pl), w_reg = (S)std::sqrt((S)p.stiffness);
  for (size_t i = 0; i < n; i++) {
    if (!(use_pt || use_pl) || corr.off[i] == corr.off[i + 1]) continue;
    S xi[6] = {0, 0, 0, 0, 0, 0}, wj_pt = 0, wr_pt = 0, wj_pl = 0, wr_pl = 0;
    const S W = ctrl.W[i];
    if (W != (S)0) {
      for (uint64_t k = ctrl.off[i]; k < ctrl.off[i + 1]; k++)
        for (int u = 0; u < 6; u++) xi[u] = xi[u] + ctrl.ws[k] * x[6 * (size_t)ctrl.sidx[k] + u];
      const S inv = (S)1 / W;
      for (int u = 0; u < 6; u++) xi[u] = xi[u] * inv;
      wr_pt = w_pt;
      wr_pl = w_pl;
      wj_pt = w_pt / W;
      wj_pl = w_pl / W;
    }
    const S s[3] = {(S)src_p[3 * i], (S)src_p[3 * i + 1], (S)src_p[3 * i + 2]};
    for (uint32_t k = corr.off[i]; k < corr.off[i + 1]; k++) {
      const size_t j = corr.dst[k];
      const S d[3] = {(S)dst_p[3 * j], (S)dst_p[3 * j + 1], (S)dst_p[3 * j + 2]};
      S nrm[3] = {0, 0, 0};
      if (use_pl)
        for (int r = 0; r < 3; r++) nrm[r] = (S)dst_n[3 * j + r];
      data_rows<S>(xi, s, d, nrm, use_pt, wj_pt, wr_pt, use_pl, wj_pl, wr_pl, &sys.B[21 * i], &sys.g[6 * i]);
    }
  }
  for (size_t j = 0; j < m; j++) {
    S* b = &sys.b[6 * j];
    S* dg = &sys.diag[6 * j];
    const auto& inc = ctrl.inc[j];
    for (size_t t = 0; t < inc.size();) {  // one group per point: (sum of its w)^2 diag(B_i)
      const uint32_t i = inc[t].first;
      S sw = 0;
      for (; t < inc.size() && inc[t].first == i; t++) {
        const S wk = ctrl.ws[inc[t].second];
        sw = sw + wk;
        for (int u = 0; u < 6; u++) b[u] = b[u] + wk * sys.g[6 * (size_t)i + u];
      }
      const S s2 = sw * sw;
      for (int u = 0; u < 6; u++) dg[u] = dg[u] + s2 * sys.B[21 * (size_t)i + upper_index(u, u)];
    }
    const S* xj = &x[6 * j];
    for (const auto& ie : arcs.inc[j]) {  // :1734-1804
      const uint32_t e = ie.first, o = ie.second;
      const bool lo = j < o;
      const S w = w_reg * (S)std::sqrt((S)std::exp((double)((S)p.reg_coeff * (S)arcs.d2[e])));
      for (int u = 0; u < 6; u++) {
        const S diff = lo ? xj[u] - x[6 * o + u] : x[6 * o + u] - xj[u];
        const S h = w * sqrt_huber_d<S>(diff, (S)p.huber);
        const S res = -(w * sqrt_huber<S>(diff, (S)p.huber));
        const S c = h * h;
        dg[u] = dg[u] + c;
        b[u] = b[u] + (lo ? h : -h) * res;
        if (lo) sys.c[6 * e + u] = c;
      }
    }
  }
}

template <class S>
void matvec_sparse(const SparseSystem<S>& sys, const Ctrl<S>& ctrl, const Arcs& arcs, const std::vector<S>& p,
                   std::vector<S>& q) {
  const size_t n = ctrl.W.size(), m = ctrl.inc.size();
  std::vector<S> y(6 * n);
  for (size_t i = 0; i < n; i++) {
    S P[6] = {0, 0, 0, 0, 0, 0};
    for (uint64_t k = ctrl.off[i]; k < ctrl.off[i + 1]; k++)
      for (int u = 0; u < 6; u++) P[u] = P[u] + ctrl.ws[k] * p[6 * (size_t)ctrl.sidx[k] + u];
    const S* B = &sys.B[21 * i];
    for (int r = 0; r < 6; r++) {
      S s = 0;
      for (int c = 0; c < 6; c++) s = s + B[r <= c ? upper_index(r, c) : upper_index(c, r)] * P[c];
      y[6 * i + r] = s;
    }
  }
  for (size_t j = 0; j < m; j++) {
    S qj[6] = {0, 0, 0, 0, 0, 0};
    for (const auto& pe : ctrl.inc[j])
      for (int u = 0; u < 6; u++) qj[u] = qj[u] + ctrl.ws[pe.second] * y[6 * (size_t)pe.first + u];
    for (const auto& ie : arcs.inc[j])
      for (int u = 0; u < 6; u++) qj[u] = qj[u] + sys.c[6 * ie.first + u] * (p[6 * j + u] - p[6 * (size_t)ie.second + u]);
    for (int u = 0; u < 6; u++) q[6 * j + u] = qj[u];
  }
}

// Eigen::ConjugateGradient as written out in warp_field_oracle.cpp, on the node unknowns
template <class S>
uint64_t cg_sparse(const SparseSystem<S>& sys, const Ctrl<S>& ctrl, const Arcs& arcs, uint64_t max_iter, double tol,
                   std::vector<S>& x, float* err) {
  const size_t mm = sys.b.size();
  x.assign(mm, (S)0);
  std::vector<S> r(sys.b), p(mm), q(mm), z(mm), inv(mm);
  for (size_t k = 0; k < mm; k++) inv[k] = sys.diag[k] != (S)0 ? (S)1 / sys.diag[k] : (S)1;
  const double rhs2 = dotd(r, r);
  *err = 0.f;
  if (rhs2 == 0.0) return 0;
  const double threshold = std::max(tol * tol * rhs2, (double)FLT_MIN);
  double rr = rhs2;
  uint64_t it = 0;
  if (!(rr < threshold)) {
    for (size_t k = 0; k < mm; k++) p[k] = inv[k] * r[k];
    double abs_new = dotd(r, p);
    while (it < max_iter) {
      matvec_sparse(sys, ctrl, arcs, p, q);
      const S alpha = (S)(abs_new / dotd(p, q));
      for (size_t k = 0; k < mm; k++) {
        x[k] = x[k] + alpha * p[k];
        r[k] = r[k] - alpha * q[k];
      }
      rr = dotd(r, r);
      if (rr < threshold) break;
      for (size_t k = 0; k < mm; k++) z[k] = inv[k] * r[k];
      const double abs_old = abs_new;
      abs_new = dotd(r, z);
      const S beta = (S)(abs_new / abs_old);
      for (size_t k = 0; k < mm; k++) p[k] = z[k] + beta * p[k];
      it++;
    }
  }
  *err = (float)std::sqrt(rr / rhs2);
  return it;
}

struct Input {
  size_t n_dst, n_src, m;
  const float *dst_p, *dst_n, *src_p;
  const uint64_t* ctrl_off;
  const int64_t* ctrl_idx;
  const float* ctrl_val;
  float ctrl_coeff;
};

template <class S>
int solve_sparse(const Input& in, size_t n_corr, const uint64_t* first, const uint64_t* second, const Arcs& arcs,
                 const Prm& p, float* T_out, float* x_out, uint64_t* stats, float* cg_err) {
  const Ctrl<S> ctrl = make_ctrl<S>(in.n_src, in.ctrl_off, in.ctrl_idx, in.ctrl_val, in.m, in.ctrl_coeff);
  const bool use_pt = n_corr > 0 && p.w_pt > 0.f, use_pl = n_corr > 0 && p.w_pl > 0.f;
  std::vector<S> x(6 * in.m, (S)0), delta;
  bool converged = false;
  uint64_t steps = 0, cg_total = 0, cg_last = 0;
  *cg_err = 0.f;
  if ((use_pt || use_pl) && in.m > 0) {  // :1427-1433
    const CorrCsr corr = corr_csr(in.n_src, n_corr, first, second);
    SparseSystem<S> sys;
    const S tol2 = (S)p.gn_tol * (S)p.gn_tol;
    for (uint64_t it = 0; it < p.max_gn_iter; it++) {
      assemble_sparse<S>(in.dst_p, in.dst_n, in.src_p, corr, ctrl, arcs, p, use_pt, use_pl, x, sys);
      cg_last = cg_sparse<S>(sys, ctrl, arcs, p.max_cg_iter, (double)p.cg_tol, delta, cg_err);
      cg_total += cg_last;
      steps++;
      S mx = 0;
      for (size_t j = 0; j < in.m; j++) {
        S sq = 0;
        for (int u = 0; u < 6; u++) {
          x[6 * j + u] = x[6 * j + u] + delta[6 * j + u];
          sq = sq + delta[6 * j + u] * delta[6 * j + u];
        }
        if (sq > mx) mx = sq;
      }
      if (mx < tol2) {
        converged = true;
        break;
      }
    }
  }
  for (size_t j = 0; j < in.m; j++) {
    double xd[6];
    for (int u = 0; u < 6; u++) xd[u] = (double)(float)x[6 * j + u];
    unknowns_to_transform(xd, T_out + 12 * j);
    if (x_out)
      for (int u = 0; u < 6; u++) x_out[6 * j + u] = (float)x[6 * j + u];
  }
  stats[0] = converged;
  stats[1] = steps;
  stats[2] = cg_total;
  stats[3] = cg_last;
  return converged;
}

}  // namespace

// estimateSparseWarpFieldCombinedMetric on the (already warped) source points: T_out [m][12] node transforms; stats =
// {converged, Gauss-Newton steps, CG iterations in total, CG iterations of the last step}; x_out [m][6] (may be NULL).
ORC_API int orc_sparse_warp_solve(size_t n_dst, const float* dst_p, const float* dst_n, size_t n_src, const float* src_p,
                                  const uint64_t* ctrl_off, const int64_t* ctrl_idx, const float* ctrl_val, size_t m,
                                  float ctrl_coeff, size_t n_corr, const uint64_t* first, const uint64_t* second,
                                  const uint64_t* reg_off, const int64_t* reg_idx, const float* reg_val, size_t n_reg,
                                  float w_pt, float w_pl, float stiffness, float huber, float reg_coeff,
                                  uint64_t max_gn_iter, float gn_tol, uint64_t max_cg_iter, float cg_tol, int use_double,
                                  float* T_out, float* x_out, uint64_t* stats, float* cg_err) {
  const Input in{n_dst, n_src, m, dst_p, dst_n, src_p, ctrl_off, ctrl_idx, ctrl_val, ctrl_coeff};
  const Arcs arcs = make_arcs(m, reg_off, reg_idx, reg_val, n_reg);
  const Prm p{w_pt, w_pl, stiffness, huber, reg_coeff, gn_tol, cg_tol, max_gn_iter, max_cg_iter};
  if (use_double) return solve_sparse<double>(in, n_corr, first, second, arcs, p, T_out, x_out, stats, cg_err);
  return solve_sparse<float>(in, n_corr, first, second, arcs, p, T_out, x_out, stats, cg_err);
}

// The normal equations in double at the node unknowns x [m][6]: b [m][6] (At b), diag [m][6] (of At At^T) and
// q [m][6] = At At^T p.
ORC_API void orc_sparse_warp_system(const float* dst_p, const float* dst_n, size_t n_src, const float* src_p,
                                    const uint64_t* ctrl_off, const int64_t* ctrl_idx, const float* ctrl_val, size_t m,
                                    float ctrl_coeff, size_t n_corr, const uint64_t* first, const uint64_t* second,
                                    const uint64_t* reg_off, const int64_t* reg_idx, const float* reg_val, size_t n_reg,
                                    float w_pt, float w_pl, float stiffness, float huber, float reg_coeff,
                                    const double* x, const double* pv, double* b, double* diag, double* q) {
  const Ctrl<double> ctrl = make_ctrl<double>(n_src, ctrl_off, ctrl_idx, ctrl_val, m, ctrl_coeff);
  const Arcs arcs = make_arcs(m, reg_off, reg_idx, reg_val, n_reg);
  const Prm p{w_pt, w_pl, stiffness, huber, reg_coeff, 0.f, 0.f, 0, 0};
  const CorrCsr corr = corr_csr(n_src, n_corr, first, second);
  std::vector<double> xv(x, x + 6 * m), pvec(pv, pv + 6 * m), qv(6 * m);
  SparseSystem<double> sys;
  assemble_sparse<double>(dst_p, dst_n, src_p, corr, ctrl, arcs, p, n_corr > 0 && w_pt > 0.f, n_corr > 0 && w_pl > 0.f,
                          xv, sys);
  matvec_sparse(sys, ctrl, arcs, pvec, qv);
  std::memcpy(b, sys.b.data(), 6 * m * sizeof(double));
  std::memcpy(diag, sys.diag.data(), 6 * m * sizeof(double));
  std::memcpy(q, qv.data(), 6 * m * sizeof(double));
}

// resampleTransforms (warp_field_utilities.hpp:14-48) in the device's float order: T_dense [n][12] from the node
// transforms T [m][12].
ORC_API void orc_sparse_warp_resample(size_t n_src, const uint64_t* ctrl_off, const int64_t* ctrl_idx,
                                      const float* ctrl_val, size_t m, float ctrl_coeff, const float* T,
                                      float* T_dense) {
  const Ctrl<float> ctrl = make_ctrl<float>(n_src, ctrl_off, ctrl_idx, ctrl_val, m, ctrl_coeff);
  for (size_t i = 0; i < n_src; i++) {
    float L[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (uint64_t k = ctrl.off[i]; k < ctrl.off[i + 1]; k++)
      for (int u = 0; u < 12; u++) L[u] = L[u] + ctrl.w[k] * T[12 * (size_t)ctrl.idx[k] + u];
    float* out = T_dense + 12 * i;
    if (ctrl.W[i] == 0.f) {
      for (int u = 0; u < 12; u++) out[u] = (u % 5 == 0) ? 1.f : 0.f;
      continue;
    }
    const float inv = 1.f / ctrl.W[i];
    M3 A;
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) A.a[r][c] = (double)(L[4 * r + c] * inv);
    const M3 R = nearest_rotation_col0_rule(A);
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) out[4 * r + c] = (float)R.a[r][c];
      out[4 * r + 3] = L[4 * r + 3] * inv;
    }
  }
}
