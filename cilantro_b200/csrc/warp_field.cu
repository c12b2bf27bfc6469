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
#include <cooperative_groups.h>

#include "cb_internal.hpp"
#include "icp_kernels.cuh"
#include "solve_core.hpp"
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

using namespace cb;
namespace cg = cooperative_groups;

namespace {
struct WarpStats;
}

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

constexpr int kBlock = 256;
constexpr int kWarps = kBlock / 32;

struct WarpStats {
  unsigned int max_delta_bits;  // max_i |delta_i|^2 (float bits; non-negative floats order as integers)
  unsigned int last_delta_bits; // max_i |dR_i - I|_F^2 + |dt_i|^2
  unsigned int num_corr;
  unsigned int cg_iters;
  float cg_err;
  unsigned int pad_;
};

__device__ __forceinline__ float fm(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fs(float a, float b) { return __fsub_rn(a, b); }

// sqrtHuberLoss / sqrtHuberLossDerivative (warp_field_estimation.hpp:10-36), float
__device__ __forceinline__ float sqrt_huber(float x, float delta) {
  const float xa = fabsf(x);
  if (xa > delta) return __fsqrt_rn(fm(delta, fs(xa, fm(0.5f, delta))));
  return fm(__fsqrt_rn(0.5f), xa);
}
__device__ __forceinline__ float sqrt_huber_d(float x, float delta) {
  const float xa = fabsf(x);
  const float v = xa > delta ? __fdiv_rn(delta, fm(2.f, __fsqrt_rn(fm(delta, fs(xa, fm(0.5f, delta))))))
                             : __fsqrt_rn(0.5f);
  return x < 0.f ? -v : v;
}

__device__ __forceinline__ float dot3(float a0, float a1, float a2, float b0, float b1, float b2) {
  return fa(fa(fm(a0, b0), fm(a1, b1)), fm(a2, b2));
}

__device__ __forceinline__ int upper_index(int r, int c) { return r * 6 - (r * (r - 1)) / 2 + (c - r); }

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

// Rows of warp_field_estimation.hpp:496-600 for one correspondence (d, n) of the source point s, linearised at the
// Euler angles (a, b, c) and translation t; J x = res per row, accumulated into B (upper) and g.
__device__ __forceinline__ void add_row(const float J[6], float res, float (&B)[21], float (&g)[6]) {
  int k = 0;
#pragma unroll
  for (int r = 0; r < 6; r++) {
#pragma unroll
    for (int c = r; c < 6; c++, k++) B[k] = fa(B[k], fm(J[r], J[c]));
    g[r] = fa(g[r], fm(J[r], res));
  }
}

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
      // computeRotationTerms (:38-89); rot = rot_coeffs^T = Rz(c) Ry(b) Rx(a)
      const float sa = (float)sin((double)x[0]), ca = (float)cos((double)x[0]);
      const float sb = (float)sin((double)x[1]), cb_ = (float)cos((double)x[1]);
      const float sc = (float)sin((double)x[2]), cc = (float)cos((double)x[2]);
      float M[3][3], Da[3][3], Db[3][3], Dc[3][3];  // the reference's (row, col) of rot_coeffs and its derivatives
      M[0][0] = fm(cc, cb_);
      M[1][0] = fa(fm(-sc, ca), fm(fm(cc, sb), sa));
      M[2][0] = fa(fm(sc, sa), fm(fm(cc, sb), ca));
      M[0][1] = fm(sc, cb_);
      M[1][1] = fa(fm(cc, ca), fm(fm(sc, sb), sa));
      M[2][1] = fa(fm(-cc, sa), fm(fm(sc, sb), ca));
      M[0][2] = -sb;
      M[1][2] = fm(cb_, sa);
      M[2][2] = fm(cb_, ca);
      Da[0][0] = 0.f;
      Da[1][0] = fa(fm(sc, sa), fm(fm(cc, sb), ca));
      Da[2][0] = fs(fm(sc, ca), fm(fm(cc, sb), sa));
      Da[0][1] = 0.f;
      Da[1][1] = fa(fm(-cc, sa), fm(fm(sc, sb), ca));
      Da[2][1] = fs(fm(-cc, ca), fm(fm(sc, sb), sa));
      Da[0][2] = 0.f;
      Da[1][2] = fm(cb_, ca);
      Da[2][2] = fm(-cb_, sa);
      Db[0][0] = fm(-cc, sb);
      Db[1][0] = fm(fm(cc, cb_), sa);
      Db[2][0] = fm(fm(cc, cb_), ca);
      Db[0][1] = fm(-sc, sb);
      Db[1][1] = fm(fm(sc, cb_), sa);
      Db[2][1] = fm(fm(sc, cb_), ca);
      Db[0][2] = -cb_;
      Db[1][2] = fm(-sb, sa);
      Db[2][2] = fm(-sb, ca);
      Dc[0][0] = fm(-sc, cb_);
      Dc[1][0] = fs(fm(-cc, ca), fm(fm(sc, sb), sa));
      Dc[2][0] = fs(fm(cc, sa), fm(fm(sc, sb), ca));
      Dc[0][1] = fm(cc, cb_);
      Dc[1][1] = fa(fm(-sc, ca), fm(fm(cc, sb), sa));
      Dc[2][1] = fa(fm(sc, sa), fm(fm(cc, sb), ca));
      Dc[0][2] = 0.f;
      Dc[1][2] = 0.f;
      Dc[2][2] = 0.f;
      const float4 s4 = a.warped[i];
      const float s[3] = {s4.x, s4.y, s4.z};
      const float d[3] = {a.dst_raw[3 * (size_t)j], a.dst_raw[3 * (size_t)j + 1], a.dst_raw[3 * (size_t)j + 2]};
      float ts[3], das[3], dbs[3], dcs[3];
#pragma unroll
      for (int r = 0; r < 3; r++) {  // (M^T s)_r = M(0,r) s0 + M(1,r) s1 + M(2,r) s2
        ts[r] = fs(d[r], fa(dot3(M[0][r], M[1][r], M[2][r], s[0], s[1], s[2]), x[3 + r]));
        das[r] = dot3(Da[0][r], Da[1][r], Da[2][r], s[0], s[1], s[2]);
        dbs[r] = dot3(Db[0][r], Db[1][r], Db[2][r], s[0], s[1], s[2]);
        dcs[r] = dot3(Dc[0][r], Dc[1][r], Dc[2][r], s[0], s[1], s[2]);
      }
      if (a.use_pt) {
        const float w = a.w_pt_sqrt;  // sqrt(w_pt) * sqrt(UnityWeightEvaluator = 1)
#pragma unroll
        for (int r = 0; r < 3; r++) {
          float J[6] = {fm(das[r], w), fm(dbs[r], w), fm(dcs[r], w), 0.f, 0.f, 0.f};
          J[3 + r] = w;
          add_row(J, fm(ts[r], w), B, g);
        }
      }
      if (a.use_pl) {
        const float w = a.w_pl_sqrt;
        const float nn[3] = {a.dst_nrm[3 * (size_t)j], a.dst_nrm[3 * (size_t)j + 1], a.dst_nrm[3 * (size_t)j + 2]};
        const float J[6] = {fm(dot3(nn[0], nn[1], nn[2], das[0], das[1], das[2]), w),
                            fm(dot3(nn[0], nn[1], nn[2], dbs[0], dbs[1], dbs[2]), w),
                            fm(dot3(nn[0], nn[1], nn[2], dcs[0], dcs[1], dcs[2]), w),
                            fm(nn[0], w), fm(nn[1], w), fm(nn[2], w)};
        add_row(J, fm(dot3(nn[0], nn[1], nn[2], ts[0], ts[1], ts[2]), w), B, g);
      }
    }
  }
  if (found) atomicAdd(&a.stats->num_corr, found);  // integer: order-free

  float diag[6];
#pragma unroll
  for (int u = 0; u < 6; u++) diag[u] = B[upper_index(u, u)];
  // regularisation (:603-673): arc (lo, hi), diff = x_lo - x_hi, entries +h' (lo) and -h' (hi), residual -w huber(diff)
  for (uint32_t k = a.inc_off[i]; k < a.inc_off[i + 1]; k++) {
    const uint32_t e = a.inc_arc[k], o = a.inc_other[k];
    const bool lo = i < o;
    const float w = fm(a.reg_sqrt, __fsqrt_rn((float)exp((double)fm(a.reg_coeff, a.arc_d2[e]))));
    float xo[6];
#pragma unroll
    for (int u = 0; u < 6; u++) xo[u] = a.xs[6 * (size_t)o + u];
#pragma unroll
    for (int u = 0; u < 6; u++) {
      const float diff = lo ? fs(x[u], xo[u]) : fs(xo[u], x[u]);
      const float h = fm(w, sqrt_huber_d(diff, a.huber));
      const float res = -fm(w, sqrt_huber(diff, a.huber));
      const float c = fm(h, h);
      diag[u] = fa(diag[u], c);
      g[u] = fa(g[u], fm(lo ? h : -h, res));
      if (lo) a.arc_c[6 * (size_t)e + u] = c;
    }
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
  uint32_t n;
  const float* B;
  const float* b;
  const float* inv;
  const uint32_t* inc_off;
  const uint32_t* inc_arc;
  const uint32_t* inc_other;
  const float* arc_c;
  float* x;
  float* r;
  float* p;
  float* z;
  float* q;
  float* xs;          // += x at the end
  double* part;       // [5][gridDim.x]
  unsigned int max_iter;
  double tol;
  WarpStats* stats;
};

// Block sum of NV values in a fixed order (warp tree, then the warps in order), stored as this block's row of
// `part` ([NV][gridDim.x]).
template <int NV>
__device__ __forceinline__ void block_partials(double (&v)[NV], double* part) {
  __shared__ double sh[NV][kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NV; k++) {
    double t = v[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xffffffffu, t, o);
    if (lane == 0) sh[k][warp] = t;
  }
  __syncthreads();
  if (threadIdx.x < NV) {
    double t = 0;
    for (int w = 0; w < kWarps; w++) t += sh[threadIdx.x][w];
    part[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = t;
  }
  __syncthreads();
}

// After a grid sync: the totals of the rows, summed in block order by warp 0 of every block (the same operations on
// the same data in every block, so every block takes the same branch).
template <int NV>
__device__ __forceinline__ void grid_totals(const double* part, double (&out)[NV]) {
  __shared__ double tot[NV];
  if (threadIdx.x < 32) {
#pragma unroll
    for (int k = 0; k < NV; k++) {
      double t = 0;
      for (unsigned int j = threadIdx.x; j < gridDim.x; j += 32) t += __ldcg(part + (size_t)k * gridDim.x + j);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xffffffffu, t, o);
      if (threadIdx.x == 0) tot[k] = t;
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < NV; k++) out[k] = tot[k];
  __syncthreads();
}

__device__ __forceinline__ void load6(const float* v, uint32_t i, float (&o)[6]) {
#pragma unroll
  for (int u = 0; u < 6; u++) o[u] = __ldcg(v + 6 * (size_t)i + u);
}
__device__ __forceinline__ void store6(float* v, uint32_t i, const float (&o)[6]) {
#pragma unroll
  for (int u = 0; u < 6; u++) v[6 * (size_t)i + u] = o[u];
}

// Eigen::ConjugateGradient with a DiagonalPreconditioner and zero initial guess (the loop written out in DESIGN
// §4.13), one Gauss-Newton step, then xs += x and the max of |x_i|^2. Cooperative launch: every block is resident.
__global__ void __launch_bounds__(kBlock) warp_cg_kernel(const CgArgs a) {
  cg::grid_group grid = cg::this_grid();
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x;
  double* const partA = a.part;                       // rr, rp of the start
  double* const partP = a.part + 2 * gridDim.x;       // p.q
  double* const partR = a.part + 3 * gridDim.x;       // rr, rz
  {
    double v[2] = {0.0, 0.0};
    for (uint32_t i = t0; i < a.n; i += stride) {
      float r[6], p[6], zero[6];
#pragma unroll
      for (int u = 0; u < 6; u++) {
        r[u] = __ldg(a.b + 6 * (size_t)i + u);
        p[u] = fm(__ldg(a.inv + 6 * (size_t)i + u), r[u]);
        zero[u] = 0.f;
      }
#pragma unroll
      for (int u = 0; u < 6; u++) {
        v[0] += (double)r[u] * (double)r[u];
        v[1] += (double)r[u] * (double)p[u];
      }
      store6(a.x, i, zero);
      store6(a.r, i, r);
      store6(a.p, i, p);
    }
    block_partials<2>(v, partA);
  }
  grid.sync();
  double tA[2];
  grid_totals<2>(partA, tA);
  __shared__ double s_rhs2;  // read again only at the end: kept out of the loop's registers
  const double rhs2 = tA[0];
  if (threadIdx.x == 0) s_rhs2 = rhs2;
  double abs_new = tA[1], rr = rhs2;
  unsigned int it = 0;
  double threshold = 0.0;
  if (rhs2 != 0.0) {
    threshold = fmax(a.tol * a.tol * rhs2, (double)FLT_MIN);
    if (!(rr < threshold)) {
      while (it < a.max_iter) {
        {  // q = A p, p.q
          double v[1] = {0.0};
          for (uint32_t i = t0; i < a.n; i += stride) {
            float p[6], q[6];
            load6(a.p, i, p);
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
              load6(a.p, o, po);
#pragma unroll
              for (int u = 0; u < 6; u++) q[u] = fa(q[u], fm(__ldg(a.arc_c + 6 * (size_t)e + u), fs(p[u], po[u])));
            }
#pragma unroll
            for (int u = 0; u < 6; u++) v[0] += (double)p[u] * (double)q[u];
            store6(a.q, i, q);
          }
          block_partials<1>(v, partP);
        }
        grid.sync();
        double tP[1];
        grid_totals<1>(partP, tP);
        const float alpha = (float)(abs_new / tP[0]);
        {  // x += alpha p, r -= alpha q, z = M^-1 r; |r|^2, r.z
          double v[2] = {0.0, 0.0};
          for (uint32_t i = t0; i < a.n; i += stride) {
            float x[6], r[6], p[6], q[6], z[6];
            load6(a.x, i, x);
            load6(a.r, i, r);
            load6(a.p, i, p);
            load6(a.q, i, q);
#pragma unroll
            for (int u = 0; u < 6; u++) {
              x[u] = fa(x[u], fm(alpha, p[u]));
              r[u] = fs(r[u], fm(alpha, q[u]));
              z[u] = fm(__ldg(a.inv + 6 * (size_t)i + u), r[u]);
              v[0] += (double)r[u] * (double)r[u];
              v[1] += (double)r[u] * (double)z[u];
            }
            store6(a.x, i, x);
            store6(a.r, i, r);
            store6(a.z, i, z);
          }
          block_partials<2>(v, partR);
        }
        grid.sync();
        double tR[2];
        grid_totals<2>(partR, tR);
        rr = tR[0];
        if (rr < threshold) break;
        const double abs_old = abs_new;
        abs_new = tR[1];
        const float beta = (float)(abs_new / abs_old);
        for (uint32_t i = t0; i < a.n; i += stride) {  // p = z + beta p
          float z[6], p[6];
          load6(a.z, i, z);
          load6(a.p, i, p);
#pragma unroll
          for (int u = 0; u < 6; u++) p[u] = fa(z[u], fm(beta, p[u]));
          store6(a.p, i, p);
        }
        it++;
        grid.sync();
      }
    }
  }
  // Gauss-Newton update (:682-693): xs += delta, max_i |delta_i|^2 (fp32, as the reference)
  float mx = 0.f;
  for (uint32_t i = t0; i < a.n; i += stride) {
    float d[6], xs[6];
    load6(a.x, i, d);
    load6(a.xs, i, xs);
    float sq = 0.f;
#pragma unroll
    for (int u = 0; u < 6; u++) {
      xs[u] = fa(xs[u], d[u]);
      sq = fa(sq, fm(d[u], d[u]));
    }
    store6(a.xs, i, xs);
    if (sq > mx) mx = sq;  // NaN never passes, as in the reference's comparison
  }
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 16));
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 8));
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 4));
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
  if ((threadIdx.x & 31) == 0 && mx > 0.f) atomicMax(&a.stats->max_delta_bits, __float_as_uint(mx));
  if (t0 == 0) {
    a.stats->cg_iters = (unsigned int)it;
    a.stats->cg_err = s_rhs2 != 0.0 ? (float)sqrt(rr / s_rhs2) : 0.f;
  }
}

// The estimator's output (:701-712) and the ICP update (icp_warp_field_combined_metric_dense.hpp updateEstimate):
// dT_i = (rotation(AngleAxis(c, Z) AngleAxis(b, Y) AngleAxis(a, X)), (tx, ty, tz)); compose: T_i <- dT_i T_i with
// its linear part projected on the rotations (TransformSet::preApply), else T_i <- dT_i. The max of
// |dR_i - I|_F^2 + |dt_i|^2, the warped points T_i s_i for the next search and the number of correspondences of the
// search (nn may be nullptr).
__global__ void warp_compose_kernel(uint32_t n, const float* __restrict__ src_raw, const float* __restrict__ xs, float* T,
                                    bool compose, float4* __restrict__ warped, const int* __restrict__ nn,
                                    WarpStats* stats) {
  float mx = 0.f;
  unsigned int found = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (nn && nn[i] >= 0) ++found;
    float x[6];
#pragma unroll
    for (int u = 0; u < 6; u++) x[u] = xs[6 * (size_t)i + u];
    const double ca = cos((double)x[0]), sa = sin((double)x[0]);
    const double cb_ = cos((double)x[1]), sb = sin((double)x[1]);
    const double cc = cos((double)x[2]), sc = sin((double)x[2]);
    la::Mat3 A;  // Rz(c) Ry(b) Rx(a)
    A.m[0][0] = cc * cb_;
    A.m[0][1] = cc * sb * sa - sc * ca;
    A.m[0][2] = cc * sb * ca + sc * sa;
    A.m[1][0] = sc * cb_;
    A.m[1][1] = sc * sb * sa + cc * ca;
    A.m[1][2] = sc * sb * ca - cc * sa;
    A.m[2][0] = -sb;
    A.m[2][1] = cb_ * sa;
    A.m[2][2] = cb_ * ca;
    const la::Mat3 R = la::nearest_rotation(A, 0);  // LinearTransform::rotation()
    float dT[12];
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) dT[r * 4 + c] = (float)R.m[r][c];
      dT[r * 4 + 3] = x[3 + r];
    }
    float sq = 0.f;  // (linear - I).squaredNorm() (column-major) + translation.squaredNorm()
    for (int c = 0; c < 3; c++)
      for (int r = 0; r < 3; r++) {
        const float e = fs(dT[r * 4 + c], r == c ? 1.f : 0.f);
        sq = fa(sq, fm(e, e));
      }
    sq = fa(sq, fa(fa(fm(x[3], x[3]), fm(x[4], x[4])), fm(x[5], x[5])));
    if (sq > mx) mx = sq;
    float Ti[12];
    if (compose) {
      for (int u = 0; u < 12; u++) Ti[u] = T[12 * (size_t)i + u];
      sc::compose(dT, Ti, Ti);
      sc::reorthonormalize(Ti);
    } else {
      for (int u = 0; u < 12; u++) Ti[u] = dT[u];
    }
    for (int u = 0; u < 12; u++) T[12 * (size_t)i + u] = Ti[u];
    if (warped) {
      const float s[3] = {src_raw[3 * (size_t)i], src_raw[3 * (size_t)i + 1], src_raw[3 * (size_t)i + 2]};
      float q[3];
      sc::apply_point(Ti, s, q);
      warped[i] = make_float4(q[0], q[1], q[2], __int_as_float((int)i));
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    found += __shfl_xor_sync(0xffffffffu, found, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (mx > 0.f) atomicMax(&stats->last_delta_bits, __float_as_uint(mx));
    if (found) atomicAdd(&stats->num_corr, found);
  }
}

// warped_i = T_i s_i (T may be nullptr: identities, which also resets T to them)
__global__ void warp_points_kernel(uint32_t n, const float* __restrict__ src_raw, float* T, bool identity,
                                   float4* __restrict__ warped) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float Ti[12];
    if (identity) {
      sc::t34_identity(Ti);
      for (int u = 0; u < 12; u++) T[12 * (size_t)i + u] = Ti[u];
    } else {
      for (int u = 0; u < 12; u++) Ti[u] = T[12 * (size_t)i + u];
    }
    const float s[3] = {src_raw[3 * (size_t)i], src_raw[3 * (size_t)i + 1], src_raw[3 * (size_t)i + 2]};
    float q[3];
    sc::apply_point(Ti, s, q);
    warped[i] = make_float4(q[0], q[1], q[2], __int_as_float((int)i));
  }
}

// incidence entries 2e (lo end) and 2e + 1 (hi end), keyed by point
__global__ void incidence_keys_kernel(const uint32_t* __restrict__ lo, const uint32_t* __restrict__ hi, uint32_t m,
                                      uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < m; e += gridDim.x * blockDim.x) {
    keys[2 * (size_t)e] = lo[e];
    vals[2 * (size_t)e] = 2 * e;
    keys[2 * (size_t)e + 1] = hi[e];
    vals[2 * (size_t)e + 1] = 2 * e + 1;
  }
}

// after the sort: arc and other end per entry, and off[p] = first entry of point p (off[n] = total)
__global__ void incidence_fill_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, uint32_t total,
                                      uint32_t n, const uint32_t* __restrict__ lo, const uint32_t* __restrict__ hi,
                                      uint32_t* __restrict__ inc_arc, uint32_t* __restrict__ inc_other,
                                      uint32_t* __restrict__ off) {
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k <= total; k += gridDim.x * blockDim.x) {
    const uint32_t cur = k < total ? (uint32_t)keys[k] : n;
    const uint32_t prev = k > 0 ? (uint32_t)keys[k - 1] : 0u;
    const uint32_t first = k > 0 ? prev + 1 : 0u;
    for (uint32_t p = first; p <= cur && p <= n; p++) off[p] = k;
    if (k < total) {
      const uint32_t e = vals[k] >> 1;
      inc_arc[k] = e;
      inc_other[k] = (vals[k] & 1u) ? lo[e] : hi[e];
    }
  }
}

int grid_for(cb_context* ctx, size_t n) {
  return (int)std::max<size_t>(1, std::min<size_t>((size_t)ctx->sm_count * 8, (n + kBlock - 1) / kBlock));
}

int check_params(const cb_warp_icp* w, const cb_warp_params* p) {
  CB_CHECK(w && p, CB_ERR_INVALID, "null argument");
  CB_CHECK(p->search_dir == CB_SECOND_TO_FIRST && p->require_reciprocal == 0 && p->one_to_one == 0 &&
               !(p->inlier_fraction > 0.0 && p->inlier_fraction < 1.0),
           CB_ERR_UNSUPPORTED, "the warp-field ICP supports the default correspondence engine only");
  CB_CHECK(!(p->w_pl > 0.f) || w->dst->d_raw_nrm, CB_ERR_INVALID,
           "w_pl > 0 needs a destination cloud with normals");
  CB_CUDA(cudaSetDevice(w->ctx->device));
  return CB_OK;
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
  ca.n = w->n;
  ca.B = w->d_B;
  ca.b = w->d_b;
  ca.inv = w->d_inv;
  ca.inc_off = w->d_inc_off;
  ca.inc_arc = w->d_inc_arc;
  ca.inc_other = w->d_inc_other;
  ca.arc_c = w->d_arc_c;
  ca.x = w->d_vec;
  ca.r = w->d_vec + 6 * n;
  ca.p = w->d_vec + 12 * n;
  ca.z = w->d_vec + 18 * n;
  ca.q = w->d_vec + 24 * n;
  ca.xs = w->d_xs;
  ca.part = w->d_part;
  ca.max_iter = (unsigned int)std::min<uint64_t>(p->max_cg_iter, 0xffffffffu);
  ca.tol = (double)p->cg_tol;
  ca.stats = (WarpStats*)w->d_stats;
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

int search(cb_warp_icp* w, float max_d2) {
  if (w->n == 0) return CB_OK;
  IcpArgs a{};
  a.dst = grid_view(w->dst);
  a.src_pts = w->d_warped;
  a.n_src = w->n;
  a.T = rigid_from_t12(nullptr);
  a.Tin = rigid_from_t12(nullptr);
  a.max_d2 = max_d2;
  a.out_idx = w->d_nn;
  a.out_d2 = w->d_nn_d2;
  return launch_icp_pass(w->ctx, a, kModeKnn, true, false, false);
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
  cudaStream_t s = ctx->stream;
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
  const uint32_t m32 = w->n_arcs, total = 2 * m32;
  if (m32) {
    CB_CUDA(cudaMemcpyAsync(w->d_arc_lo, lo.data(), m32 * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CB_CUDA(cudaMemcpyAsync(w->d_arc_hi, hi.data(), m32 * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CB_CUDA(cudaMemcpyAsync(w->d_arc_d2, d2.data(), m32 * sizeof(float), cudaMemcpyHostToDevice, s));
  }
  DeviceScope scope(ctx);
  uint64_t *keys = nullptr, *keys_tmp = nullptr;
  uint32_t *vals = nullptr, *vals_tmp = nullptr;
  CB_TRY(scope.alloc(&keys, total));
  CB_TRY(scope.alloc(&keys_tmp, total));
  CB_TRY(scope.alloc(&vals, total));
  CB_TRY(scope.alloc(&vals_tmp, total));
  if (m32) {
    incidence_keys_kernel<<<grid_for(ctx, m32), kBlock, 0, s>>>(w->d_arc_lo, w->d_arc_hi, m32, keys, vals);
    ctx->launches += 1;
    CB_CUDA(cudaGetLastError());
    int bits = 1;
    while (bits < 32 && (1ull << bits) < (uint64_t)nn) bits++;
    CB_TRY(radix_sort_pairs_u64(ctx, keys, vals, keys_tmp, vals_tmp, total, bits));
  }
  incidence_fill_kernel<<<grid_for(ctx, (size_t)total + 1), kBlock, 0, s>>>(keys, vals, total, n, w->d_arc_lo,
                                                                           w->d_arc_hi, w->d_inc_arc, w->d_inc_other,
                                                                           w->d_inc_off);
  ctx->launches += 1;
  CB_CUDA(cudaGetLastError());
  CB_CUDA(cudaStreamSynchronize(s));
  return CB_OK;
}

int cb_warp_icp_create(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src, const uint64_t* reg_offsets,
                       const int64_t* reg_index, const float* reg_value, size_t n_reg, cb_warp_icp** out) {
  CB_CHECK(ctx && dst && src && out, CB_ERR_INVALID, "null argument");
  CB_CHECK(dst->ctx == ctx && src->ctx == ctx, CB_ERR_INVALID, "cloud belongs to another context");
  CB_CHECK(dst->index_offset == 0 && src->index_offset == 0, CB_ERR_UNSUPPORTED,
           "the warp-field ICP runs on whole clouds (index_offset must be 0)");
  CB_CHECK(ctx->world == 1, CB_ERR_UNSUPPORTED, "the warp-field ICP runs on one rank");
  // point indices travel as signed 32-bit values: the search's matches (int), the warped points' index bits and the
  // correspondence slots
  CB_CHECK(dst->n < 0x7fffffffull && src->n < 0x7fffffffull, CB_ERR_UNSUPPORTED,
           "the warp-field ICP supports fewer than 2^31 - 1 points per cloud");
  CB_CHECK(n_reg == 0 || reg_offsets, CB_ERR_INVALID, "null neighbourhood offsets");
  const uint32_t n = (uint32_t)src->n;
  // validate the neighbourhoods and list the arcs in the reference's equation order (:410-421, :605-617)
  std::vector<uint32_t> lo, hi;
  std::vector<float> d2;
  if (n_reg) {
    CB_CHECK(reg_offsets[0] == 0, CB_ERR_INVALID, "neighbourhood offsets must start at 0");
    const uint64_t total = reg_offsets[n_reg];
    CB_CHECK(total == 0 || (reg_index && reg_value), CB_ERR_INVALID, "null neighbourhood index / value");
    for (size_t j = 0; j < n_reg; j++) {
      const uint64_t b = reg_offsets[j], e = reg_offsets[j + 1];
      CB_CHECK(b <= e && e <= total, CB_ERR_INVALID, "neighbourhood offsets must be non-decreasing");
      for (uint64_t k = b; k < e; k++)
        CB_CHECK(reg_index[k] >= 0 && (uint64_t)reg_index[k] < n, CB_ERR_INVALID,
                 "neighbourhood index outside the source cloud");
      if (e - b < 2) continue;
      const uint32_t c = (uint32_t)reg_index[b];
      for (uint64_t k = b + 1; k < e; k++) {
        const uint32_t o = (uint32_t)reg_index[k];
        if (o == c) continue;  // self-arc: its two entries cancel
        lo.push_back(std::min(c, o));
        hi.push_back(std::max(c, o));
        d2.push_back(reg_value[k]);
      }
    }
  }
  CB_CHECK(lo.size() < 0x7fffffffull, CB_ERR_UNSUPPORTED, "too many regularisation arcs (2^31 - 1 at most)");
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
    CB_TRY(search(w, p->max_d2));  // updateCorrespondences
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
  // correspondence slots grouped by source point, list order kept within a point
  std::vector<uint32_t> off((size_t)w->n + 1, 0u);
  for (size_t c = 0; c < n_corr; c++) {
    CB_CHECK(corr_first[c] < w->dst->n && corr_second[c] < w->n, CB_ERR_INVALID, "correspondence index out of range");
    off[corr_second[c] + 1]++;
  }
  for (size_t i = 0; i < w->n; i++) off[i + 1] += off[i];
  std::vector<int> slot(std::max<size_t>(n_corr, 1));  // dst indices < 2^31 - 1 (cb_warp_icp_create)
  {
    std::vector<uint32_t> fill(off.begin(), off.end() - 1);
    for (size_t c = 0; c < n_corr; c++) slot[fill[corr_second[c]]++] = (int)corr_first[c];
  }
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
  cb_context* ctx = w->ctx;
  CB_TRY(warp_points(w, T));
  DeviceScope scope(ctx);
  float* d_out = nullptr;
  CB_TRY(scope.alloc(&d_out, w->n));
  const bool normals = w->dst->d_raw_nrm != nullptr;
  // the combined residual reads the destination normals; without them (w_pl <= 0 here) it is w_pt |d - p|^2
  CB_TRY(launch_residuals(ctx, grid_view(w->dst), w->d_warped, nullptr, w->n, rigid_from_t12(nullptr),
                          normals ? CB_ICP_COMBINED : CB_ICP_POINT_TO_POINT, p->w_pt, p->w_pl, d_out));
  CB_CUDA(cudaMemcpyAsync(out, d_out, w->n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  if (!normals)
    for (size_t i = 0; i < w->n; i++) out[i] = p->w_pt * out[i];
  return CB_OK;
}

int cb_warp_icp_correspondences(cb_warp_icp* w, uint64_t* index_first, uint64_t* index_second, float* value,
                                size_t* count) {
  CB_CHECK(w && count, CB_ERR_INVALID, "null argument");
  CB_CHECK(w->have_corr, CB_ERR_INVALID, "no estimate() has run");
  CB_CUDA(cudaSetDevice(w->ctx->device));
  std::vector<int> idx(w->n);
  std::vector<float> d2(w->n);
  if (w->n) {
    CB_CUDA(cudaMemcpyAsync(idx.data(), w->d_nn, w->n * sizeof(int), cudaMemcpyDeviceToHost, w->ctx->stream));
    CB_CUDA(cudaMemcpyAsync(d2.data(), w->d_nn_d2, w->n * sizeof(float), cudaMemcpyDeviceToHost, w->ctx->stream));
  }
  CB_CUDA(cudaStreamSynchronize(w->ctx->stream));
  size_t k = 0;
  for (size_t i = 0; i < w->n; i++) {
    if (idx[i] < 0) continue;
    if (index_first) index_first[k] = (uint64_t)idx[i];
    if (index_second) index_second[k] = i;
    if (value) value[k] = d2[i];
    ++k;
  }
  *count = k;
  return CB_OK;
}

}  // extern "C"
