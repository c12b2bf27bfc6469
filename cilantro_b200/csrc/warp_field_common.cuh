// Device and host pieces shared by the dense (warp_field.cu, DESIGN §4.13) and the sparse (sparse_warp_field.cu,
// DESIGN §4.14) rigid warp-field ICP: the Huber rules, the rotation terms and data rows of the estimators, the block
// and grid partial sums, the preconditioned CG loop, the compose step, the arc incidence and the 1-NN search on the
// warped points; on the host the object core both objects build on, their creation, checks and correspondence
// uploads, the Gauss-Newton driver and the update step. Product code (sm_90a).
//
// Arithmetic: fp32 with every operation rounded on its own (no FMA contraction) wherever the oracles restate the
// order; dot products and norms in fp64, summed in a fixed order; no float atomics.
#pragma once
#include <cooperative_groups.h>

#include "cb_internal.hpp"
#include "icp_kernels.cuh"
#include "solve_core.hpp"
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>

namespace {

namespace cg = cooperative_groups;
using namespace cb;

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

// J x = res per row, accumulated into B (upper) and g.
__device__ __forceinline__ void add_row(const float J[6], float res, float (&B)[21], float (&g)[6]) {
  int k = 0;
#pragma unroll
  for (int r = 0; r < 6; r++) {
#pragma unroll
    for (int c = r; c < 6; c++, k++) B[k] = fa(B[k], fm(J[r], J[c]));
    g[r] = fa(g[r], fm(J[r], res));
  }
}

// Rows of one correspondence (d, n) = destination point j of the source point s, linearised at the Euler angles
// (x0, x1, x2) and translation (x3, x4, x5): warp_field_estimation.hpp:496-600 (dense) and :1568-1731 (sparse). The
// Jacobian entries of the point-to-point (3 rows) and point-to-plane (1 row) terms are scaled by wj_pt / wj_pl, their
// residuals by wr_pt / wr_pl; accumulated into B (upper) and g.
__device__ __forceinline__ void add_data_rows(const float (&x)[6], const float (&s)[3], const float* dst_raw,
                                              const float* dst_nrm, int j, bool use_pt, bool use_pl, float wj_pt,
                                              float wr_pt, float wj_pl, float wr_pl, float (&B)[21], float (&g)[6]) {
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
  const float d[3] = {dst_raw[3 * (size_t)j], dst_raw[3 * (size_t)j + 1], dst_raw[3 * (size_t)j + 2]};
  float ts[3], das[3], dbs[3], dcs[3];
#pragma unroll
  for (int r = 0; r < 3; r++) {  // (M^T s)_r = M(0,r) s0 + M(1,r) s1 + M(2,r) s2
    ts[r] = fs(d[r], fa(dot3(M[0][r], M[1][r], M[2][r], s[0], s[1], s[2]), x[3 + r]));
    das[r] = dot3(Da[0][r], Da[1][r], Da[2][r], s[0], s[1], s[2]);
    dbs[r] = dot3(Db[0][r], Db[1][r], Db[2][r], s[0], s[1], s[2]);
    dcs[r] = dot3(Dc[0][r], Dc[1][r], Dc[2][r], s[0], s[1], s[2]);
  }
  if (use_pt) {
#pragma unroll
    for (int r = 0; r < 3; r++) {
      float J[6] = {fm(das[r], wj_pt), fm(dbs[r], wj_pt), fm(dcs[r], wj_pt), 0.f, 0.f, 0.f};
      J[3 + r] = wj_pt;
      add_row(J, fm(ts[r], wr_pt), B, g);
    }
  }
  if (use_pl) {
    const float nn[3] = {dst_nrm[3 * (size_t)j], dst_nrm[3 * (size_t)j + 1], dst_nrm[3 * (size_t)j + 2]};
    const float J[6] = {fm(dot3(nn[0], nn[1], nn[2], das[0], das[1], das[2]), wj_pl),
                        fm(dot3(nn[0], nn[1], nn[2], dbs[0], dbs[1], dbs[2]), wj_pl),
                        fm(dot3(nn[0], nn[1], nn[2], dcs[0], dcs[1], dcs[2]), wj_pl),
                        fm(nn[0], wj_pl), fm(nn[1], wj_pl), fm(nn[2], wj_pl)};
    add_row(J, fm(dot3(nn[0], nn[1], nn[2], ts[0], ts[1], ts[2]), wr_pl), B, g);
  }
}

// One Huber regularisation arc seen from one end (:603-673, :1734-1804): diff = x_lo - x_hi, entries +h' (lo) and
// -h' (hi), residual -w huber(diff). Adds c = h'^2 to diag and the arc's share to g; returns c per unknown in c_out.
__device__ __forceinline__ void add_arc(const float (&x)[6], const float (&xo)[6], bool lo, float w, float huber,
                                        float (&diag)[6], float (&g)[6], float (&c_out)[6]) {
#pragma unroll
  for (int u = 0; u < 6; u++) {
    const float diff = lo ? fs(x[u], xo[u]) : fs(xo[u], x[u]);
    const float h = fm(w, sqrt_huber_d(diff, huber));
    const float res = -fm(w, sqrt_huber(diff, huber));
    const float c = fm(h, h);
    diag[u] = fa(diag[u], c);
    g[u] = fa(g[u], fm(lo ? h : -h, res));
    c_out[u] = c;
  }
}

// sqrt(stiffness) sqrt(RBFKernelWeightEvaluator(d2)) of an arc
__device__ __forceinline__ float arc_weight(float reg_sqrt, float reg_coeff, float d2) {
  return fm(reg_sqrt, __fsqrt_rn((float)exp((double)fm(reg_coeff, d2))));
}

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

// The CG vectors over n blocks of 6 unknowns.
struct CgVecs {
  uint32_t n;
  const float* b;
  const float* inv;
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

// Eigen::ConjugateGradient with a DiagonalPreconditioner and zero initial guess (the loop written out in DESIGN
// §4.13), one Gauss-Newton step, then xs += x and the max of |x_i|^2. Cooperative launch: every block is resident.
// matvec() writes q = A p for all blocks and returns this thread's fp64 partial of p.q, summed over its blocks in
// grid-stride order; it may use grid syncs of its own.
template <class MatVec>
__device__ __forceinline__ void pcg(const CgVecs& a, cg::grid_group& grid, MatVec&& matvec) {
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
          double v[1] = {matvec()};
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
  // Gauss-Newton update (:682-693, :1814-1829): xs += delta, max_i |delta_i|^2 (fp32, as the reference)
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

// The estimator's output (:701-712, :1832-1843) and the ICP update (updateEstimate of both ICP classes):
// dT_i = (rotation(AngleAxis(c, Z) AngleAxis(b, Y) AngleAxis(a, X)), (tx, ty, tz)); compose: T_i <- dT_i T_i with
// its linear part projected on the rotations (TransformSet::preApply), else T_i <- dT_i. The max of
// |dR_i - I|_F^2 + |dt_i|^2, the warped points T_i s_i for the next search (warped may be nullptr) and the number of
// correspondences of the search (nn may be nullptr).
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

// warped_i = T_i s_i (identity: T is reset to identities first)
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

// Entry k (0 <= k <= total) of an incidence sorted by key (keys < n): off[p] = k for the keys p whose entries start
// at k, so that off[p] = first entry of key p and off[n] = total.
__device__ __forceinline__ void incidence_offsets(const uint64_t* __restrict__ keys, uint32_t k, uint32_t total,
                                                  uint32_t n, uint32_t* __restrict__ off) {
  const uint32_t cur = k < total ? (uint32_t)keys[k] : n;
  const uint32_t first = k > 0 ? (uint32_t)keys[k - 1] + 1 : 0u;
  for (uint32_t p = first; p <= cur && p <= n; p++) off[p] = k;
}

// after the sort: arc and other end per entry, and off[p] = first entry of point p (off[n] = total)
__global__ void incidence_fill_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, uint32_t total,
                                      uint32_t n, const uint32_t* __restrict__ lo, const uint32_t* __restrict__ hi,
                                      uint32_t* __restrict__ inc_arc, uint32_t* __restrict__ inc_other,
                                      uint32_t* __restrict__ off) {
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k <= total; k += gridDim.x * blockDim.x) {
    incidence_offsets(keys, k, total, n, off);
    if (k < total) {
      const uint32_t e = vals[k] >> 1;
      inc_arc[k] = e;
      inc_other[k] = (vals[k] & 1u) ? lo[e] : hi[e];
    }
  }
}

// What both warp-field ICP objects hold (cb_warp_icp is this core; cb_sparse_warp_icp adds its control lists). The
// unknowns come in m blocks of 6: one block per source point (dense, m = n) or per control node (sparse).
struct WarpCore {
  explicit WarpCore(cb_context* c) : ctx(c), mem(c) {}
  cb_context* ctx = nullptr;
  DeviceScope mem;  // every buffer of the object (device and pinned host)
  const cb_cloud* dst = nullptr;
  const cb_cloud* src = nullptr;
  uint32_t n = 0;       // source points
  uint32_t m = 0;       // unknown blocks
  uint32_t n_arcs = 0;  // regularisation arcs between blocks (self-arcs dropped)
  // arcs (lo < hi) and their incidence, sorted stably by block: entries inc_off[j] .. inc_off[j+1]-1 of block j
  uint32_t* d_arc_lo = nullptr;
  uint32_t* d_arc_hi = nullptr;
  float* d_arc_d2 = nullptr;
  float* d_arc_c = nullptr;  // [n_arcs][6] c_e of the current step
  uint32_t* d_inc_off = nullptr;
  uint32_t* d_inc_arc = nullptr;
  uint32_t* d_inc_other = nullptr;
  // per block
  float* d_T = nullptr;    // [m][12] current transforms
  float* d_xs = nullptr;   // [m][6] unknowns of the running estimator call
  float* d_b = nullptr;    // [m][6] right-hand side At b
  float* d_inv = nullptr;  // [m][6] Jacobi preconditioner
  float* d_vec = nullptr;  // [5][m][6] CG vectors x, r, p, z, q
  // per point
  float* d_B = nullptr;        // [n][21] data block, upper triangle row-major
  float4* d_warped = nullptr;  // T_i s_i, .w = index bits (the search's query layout)
  int* d_nn = nullptr;         // [n] last search: dst index or -1
  float* d_nn_d2 = nullptr;
  double* d_part = nullptr;  // CG reduction partials [5][cg_grid]
  WarpStats* d_stats = nullptr;
  WarpStats* h_stats = nullptr;  // pinned
  int cg_grid = 0;
  bool have_corr = false;
};

int grid_for(cb_context* ctx, size_t n) {
  return (int)std::max<size_t>(1, std::min<size_t>((size_t)ctx->sm_count * 8, (n + kBlock - 1) / kBlock));
}

int check_params(const WarpCore* w, const cb_warp_params* p) {
  CB_CHECK(w && p, CB_ERR_INVALID, "null argument");
  CB_CHECK(p->search_dir == CB_SECOND_TO_FIRST && p->require_reciprocal == 0 && p->one_to_one == 0 &&
               !(p->inlier_fraction > 0.0 && p->inlier_fraction < 1.0),
           CB_ERR_UNSUPPORTED, "the warp-field ICP supports the default correspondence engine only");
  CB_CHECK(!(p->w_pl > 0.f) || w->dst->d_raw_nrm, CB_ERR_INVALID, "w_pl > 0 needs a destination cloud with normals");
  CB_CUDA(cudaSetDevice(w->ctx->device));
  return CB_OK;
}

// The checks both warp-field ICP objects make on their clouds and context at creation.
int check_warp_clouds(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src) {
  CB_CHECK(dst->ctx == ctx && src->ctx == ctx, CB_ERR_INVALID, "cloud belongs to another context");
  CB_CHECK(dst->index_offset == 0 && src->index_offset == 0, CB_ERR_UNSUPPORTED,
           "the warp-field ICP runs on whole clouds (index_offset must be 0)");
  CB_CHECK(ctx->world == 1, CB_ERR_UNSUPPORTED, "the warp-field ICP runs on one rank");
  // point indices travel as signed 32-bit values: the search's matches (int), the warped points' index bits and the
  // correspondence slots
  CB_CHECK(dst->n < 0x7fffffffull && src->n < 0x7fffffffull, CB_ERR_UNSUPPORTED,
           "the warp-field ICP supports fewer than 2^31 - 1 points per cloud");
  return CB_OK;
}

// Validates regularisation neighbourhoods over n_nodes unknown blocks and lists their arcs in the reference's equation
// order (:410-421, :605-617, :1472-1483): list N gives (N[0], N[j]) for j >= 1; empty lists and self-arcs give none.
int build_arcs(uint32_t n_nodes, const uint64_t* reg_offsets, const int64_t* reg_index, const float* reg_value,
               size_t n_reg, std::vector<uint32_t>& lo, std::vector<uint32_t>& hi, std::vector<float>& d2) {
  CB_CHECK(n_reg == 0 || reg_offsets, CB_ERR_INVALID, "null neighbourhood offsets");
  if (n_reg) {
    CB_CHECK(reg_offsets[0] == 0, CB_ERR_INVALID, "neighbourhood offsets must start at 0");
    const uint64_t total = reg_offsets[n_reg];
    CB_CHECK(total == 0 || (reg_index && reg_value), CB_ERR_INVALID, "null neighbourhood index / value");
    for (size_t j = 0; j < n_reg; j++) {
      const uint64_t b = reg_offsets[j], e = reg_offsets[j + 1];
      CB_CHECK(b <= e && e <= total, CB_ERR_INVALID, "neighbourhood offsets must be non-decreasing");
      for (uint64_t k = b; k < e; k++)
        CB_CHECK(reg_index[k] >= 0 && (uint64_t)reg_index[k] < n_nodes, CB_ERR_INVALID,
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
  return CB_OK;
}

// A new object on validated inputs: the destination's grid index, the core's sizes, then init(w), which allocates and
// uploads; the object is freed again when a step fails.
template <class Obj, class Init>
int create_object(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src, uint32_t m, uint32_t n_arcs, Obj** out,
                  Init&& init) {
  CB_CUDA(cudaSetDevice(ctx->device));
  CB_TRY(ensure_index(const_cast<cb_cloud*>(dst)));
  std::unique_ptr<Obj> w(new Obj(ctx));
  w->dst = dst;
  w->src = src;
  w->n = (uint32_t)src->n;
  w->m = m;
  w->n_arcs = n_arcs;
  CB_TRY(init(w.get()));
  *out = w.release();
  return CB_OK;
}

template <class Obj>
void destroy_object(Obj* w) {
  if (!w) return;
  cudaSetDevice(w->ctx->device);
  cudaStreamSynchronize(w->ctx->stream);
  delete w;
}

// The core's buffers. The cooperative grid of cg_kernel: every block resident (occupancy API), no more blocks than
// its grid-stride loops over loop_len entries need.
int alloc_core(WarpCore* w, const void* cg_kernel, size_t loop_len) {
  const size_t nn = std::max<size_t>(w->n, 1), mm = std::max<size_t>(w->m, 1), aa = std::max<size_t>(w->n_arcs, 1);
  CB_TRY(w->mem.alloc(&w->d_arc_lo, aa));
  CB_TRY(w->mem.alloc(&w->d_arc_hi, aa));
  CB_TRY(w->mem.alloc(&w->d_arc_d2, aa));
  CB_TRY(w->mem.alloc(&w->d_arc_c, 6 * aa));
  CB_TRY(w->mem.alloc(&w->d_inc_off, mm + 1));
  CB_TRY(w->mem.alloc(&w->d_inc_arc, 2 * aa));
  CB_TRY(w->mem.alloc(&w->d_inc_other, 2 * aa));
  CB_TRY(w->mem.alloc(&w->d_T, 12 * mm));
  CB_TRY(w->mem.alloc(&w->d_xs, 6 * mm));
  CB_TRY(w->mem.alloc(&w->d_b, 6 * mm));
  CB_TRY(w->mem.alloc(&w->d_inv, 6 * mm));
  CB_TRY(w->mem.alloc(&w->d_vec, 30 * mm));
  CB_TRY(w->mem.alloc(&w->d_B, 21 * nn));
  CB_TRY(w->mem.alloc(&w->d_warped, nn));
  CB_TRY(w->mem.alloc(&w->d_nn, nn));
  CB_TRY(w->mem.alloc(&w->d_nn_d2, nn));
  CB_TRY(w->mem.alloc(&w->d_stats, 1));
  CB_TRY(w->mem.alloc_host(&w->h_stats, 1));
  int per_sm = 0;
  CB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, cg_kernel, kBlock, 0));
  CB_CHECK(per_sm >= 1, CB_ERR_CUDA, "the CG kernel cannot be resident");
  w->cg_grid = (int)std::max<size_t>(
      1, std::min<size_t>((size_t)w->ctx->sm_count * per_sm, (std::max<size_t>(loop_len, 1) + kBlock - 1) / kBlock));
  return w->mem.alloc(&w->d_part, 5 * (size_t)w->cg_grid);
}

// Uploads the arcs (lo, hi, d2) and builds their incidence over the m blocks, sorted stably by block: entries
// inc_off[j] .. inc_off[j+1]-1 of block j, ascending arc. Synchronises the stream.
int upload_arc_incidence(WarpCore* w, const std::vector<uint32_t>& lo, const std::vector<uint32_t>& hi,
                         const std::vector<float>& d2) {
  cb_context* ctx = w->ctx;
  cudaStream_t s = ctx->stream;
  const uint32_t n_nodes = w->m, m32 = (uint32_t)lo.size(), total = 2 * m32;
  uint32_t *d_lo = w->d_arc_lo, *d_hi = w->d_arc_hi;
  if (m32) {
    CB_CUDA(cudaMemcpyAsync(d_lo, lo.data(), m32 * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CB_CUDA(cudaMemcpyAsync(d_hi, hi.data(), m32 * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
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
    incidence_keys_kernel<<<grid_for(ctx, m32), kBlock, 0, s>>>(d_lo, d_hi, m32, keys, vals);
    ctx->launches += 1;
    CB_CUDA(cudaGetLastError());
    int bits = 1;
    while (bits < 32 && (1ull << bits) < (uint64_t)std::max<uint32_t>(n_nodes, 1)) bits++;
    CB_TRY(radix_sort_pairs_u64(ctx, keys, vals, keys_tmp, vals_tmp, total, bits));
  }
  incidence_fill_kernel<<<grid_for(ctx, (size_t)total + 1), kBlock, 0, s>>>(keys, vals, total, n_nodes, d_lo, d_hi,
                                                                           w->d_inc_arc, w->d_inc_other, w->d_inc_off);
  ctx->launches += 1;
  CB_CUDA(cudaGetLastError());
  CB_CUDA(cudaStreamSynchronize(s));
  return CB_OK;
}

// The grid 1-NN of the ICP pass kernel on the warped points: nn[i] = destination index within max_d2, or -1.
int warp_search(const WarpCore* w, float max_d2) {
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

// computeResiduals() of both warp-field ICP classes on the warped points (see cb_warp_icp_residuals).
int warp_residuals(const WarpCore* w, const cb_warp_params* p, float* out) {
  cb_context* ctx = w->ctx;
  const uint32_t n = w->n;
  DeviceScope scope(ctx);
  float* d_out = nullptr;
  CB_TRY(scope.alloc(&d_out, n));
  const bool normals = w->dst->d_raw_nrm != nullptr;
  // the combined residual reads the destination normals; without them (w_pl <= 0 here) it is w_pt |d - p|^2
  CB_TRY(launch_residuals(ctx, grid_view(w->dst), w->d_warped, nullptr, n, rigid_from_t12(nullptr),
                          normals ? CB_ICP_COMBINED : CB_ICP_POINT_TO_POINT, p->w_pt, p->w_pl, d_out));
  CB_CUDA(cudaMemcpyAsync(out, d_out, n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  if (!normals)
    for (size_t i = 0; i < n; i++) out[i] = p->w_pt * out[i];
  return CB_OK;
}

// getCorrespondences() from the last search of estimate() (nn, nn_d2 on the device): ascending source index
int warp_correspondences(const WarpCore* w, uint64_t* index_first, uint64_t* index_second, float* value,
                         size_t* count) {
  CB_CHECK(w && count, CB_ERR_INVALID, "null argument");
  CB_CHECK(w->have_corr, CB_ERR_INVALID, "no estimate() has run");
  cb_context* ctx = w->ctx;
  const uint32_t n = w->n;
  CB_CUDA(cudaSetDevice(ctx->device));
  std::vector<int> idx(n);
  std::vector<float> d2(n);
  if (n) {
    CB_CUDA(cudaMemcpyAsync(idx.data(), w->d_nn, n * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaMemcpyAsync(d2.data(), w->d_nn_d2, n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  }
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  size_t k = 0;
  for (size_t i = 0; i < n; i++) {
    if (idx[i] < 0) continue;
    if (index_first) index_first[k] = (uint64_t)idx[i];
    if (index_second) index_second[k] = i;
    if (value) value[k] = d2[i];
    ++k;
  }
  *count = k;
  return CB_OK;
}

// Caller-supplied correspondences grouped by source point (list order kept within a point): the slot CSR the
// estimators' assembly reads (d_off[i] .. d_off[i+1]-1: the dst indices of point i), on the device for one call.
struct CorrSlots {
  explicit CorrSlots(cb_context* ctx) : scope(ctx) {}
  DeviceScope scope;
  std::vector<uint32_t> off;  // the host copies, kept until the call ends
  std::vector<int> slot;
  uint32_t* d_off = nullptr;
  int* d_slot = nullptr;
};

// Validates the indices and uploads the slots.
int upload_corr_slots(const WarpCore* w, const uint64_t* corr_first, const uint64_t* corr_second, size_t n_corr,
                      CorrSlots* cs) {
  const size_t n_dst = w->dst->n, n_src = w->n;
  std::vector<uint32_t>& off = cs->off;
  off.assign(n_src + 1, 0u);
  for (size_t c = 0; c < n_corr; c++) {
    CB_CHECK(corr_first[c] < n_dst && corr_second[c] < n_src, CB_ERR_INVALID, "correspondence index out of range");
    off[corr_second[c] + 1]++;
  }
  for (size_t i = 0; i < n_src; i++) off[i + 1] += off[i];
  cs->slot.assign(std::max<size_t>(n_corr, 1), 0);  // dst indices < 2^31 - 1 (checked at creation)
  std::vector<uint32_t> fill(off.begin(), off.end() - 1);
  for (size_t c = 0; c < n_corr; c++) cs->slot[fill[corr_second[c]]++] = (int)corr_first[c];
  CB_TRY(cs->scope.alloc(&cs->d_off, off.size()));
  CB_TRY(cs->scope.alloc(&cs->d_slot, cs->slot.size()));
  cudaStream_t s = w->ctx->stream;
  CB_CUDA(cudaMemcpyAsync(cs->d_off, off.data(), off.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
  CB_CUDA(cudaMemcpyAsync(cs->d_slot, cs->slot.data(), cs->slot.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  return CB_OK;
}

// T <- T_host ([n][12], identities when NULL; T one transform per source point) and warped_i = T_i s_i.
int warp_points(WarpCore* w, float* T, const float* T_host) {
  cb_context* ctx = w->ctx;
  if (w->n == 0) return CB_OK;
  if (T_host)
    CB_CUDA(cudaMemcpyAsync(T, T_host, 12 * (size_t)w->n * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  warp_points_kernel<<<grid_for(ctx, w->n), kBlock, 0, ctx->stream>>>(w->n, w->src->d_raw, T, T_host == nullptr,
                                                                      w->d_warped);
  ctx->launches += 1;
  CB_CUDA(cudaGetLastError());
  return CB_OK;
}

// What Gauss-Newton calls report: the flag of the last call, the steps and CG iterations summed over the calls, and
// the last step's CG iterations and error.
struct GnCounts {
  int converged = 0;
  uint64_t steps = 0, cg_total = 0, cg_last = 0;
  float cg_err = 0.f;
};

// Device times of the Gauss-Newton steps, summed: the assembly launches and the CG launch.
struct StepTimer {
  ScopedEvents ev;  // ev.e0: assembly start, ev.e1: CG start
  ScopedEvents end;  // end.e1: CG end
  double assemble = 0, cg = 0;
  int create() {
    CB_TRY(ev.create());
    return end.create();
  }
};

// One estimator call (estimateDenseWarpFieldCombinedMetric, :368-715, or estimateSparseWarpFieldCombinedMetric,
// :1388-1846) on the current warped points and correspondences: the unknowns start at zero (:460-461, :1531-1532) and
// without a data term or a correspondence it returns before any step (:398-408, :1427-1433; no_corr: the caller
// knows the list is empty, else the first step's assembly counts it). Per step, assemble() launches the caller's
// assembly of b, inv and arc_c, then the cooperative cg_kernel(ca) runs the CG over the m blocks (ca.v is filled
// here) and adds the solution to xs. timer, when given, takes the times of both.
template <class CgArgs, class Assemble>
int gauss_newton(WarpCore* w, const cb_warp_params* p, bool no_corr, Assemble&& assemble, const void* cg_kernel,
                 CgArgs& ca, GnCounts* gn, StepTimer* timer) {
  cb_context* ctx = w->ctx;
  const size_t m = w->m;
  gn->converged = 0;
  CB_CUDA(cudaMemsetAsync(w->d_xs, 0, 6 * std::max<size_t>(m, 1) * sizeof(float), ctx->stream));
  if ((!(p->w_pt > 0.f) && !(p->w_pl > 0.f)) || no_corr || w->n == 0 || m == 0) return CB_OK;
  ca.v.n = w->m;
  ca.v.b = w->d_b;
  ca.v.inv = w->d_inv;
  ca.v.x = w->d_vec;
  ca.v.r = w->d_vec + 6 * m;
  ca.v.p = w->d_vec + 12 * m;
  ca.v.z = w->d_vec + 18 * m;
  ca.v.q = w->d_vec + 24 * m;
  ca.v.xs = w->d_xs;
  ca.v.part = w->d_part;
  ca.v.max_iter = (unsigned int)std::min<uint64_t>(p->max_cg_iter, 0xffffffffu);
  ca.v.tol = (double)p->cg_tol;
  ca.v.stats = w->d_stats;
  const WarpStats* hs = w->h_stats;
  const float tol2 = p->gn_tol * p->gn_tol;
  for (uint64_t step = 0; step < p->max_gn_iter; step++) {
    CB_CUDA(cudaMemsetAsync(w->d_stats, 0, sizeof(WarpStats), ctx->stream));
    if (timer) CB_CUDA(cudaEventRecord(timer->ev.e0, ctx->stream));
    CB_TRY(assemble());
    if (timer) CB_CUDA(cudaEventRecord(timer->ev.e1, ctx->stream));
    void* args[] = {&ca};
    CB_CUDA(cudaLaunchCooperativeKernel(cg_kernel, dim3(w->cg_grid), dim3(kBlock), args, 0, ctx->stream));
    if (timer) CB_CUDA(cudaEventRecord(timer->end.e1, ctx->stream));
    ctx->launches += 1;
    CB_CUDA(cudaMemcpyAsync(w->h_stats, w->d_stats, sizeof(WarpStats), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    if (timer) {
      float ta = 0.f, tc = 0.f;
      CB_CUDA(cudaEventElapsedTime(&ta, timer->ev.e0, timer->ev.e1));
      CB_CUDA(cudaEventElapsedTime(&tc, timer->ev.e1, timer->end.e1));
      timer->assemble += ta;
      timer->cg += tc;
    }
    // no correspondence: b = 0, so the step left xs at zero; the reference returns before any step
    if (step == 0 && hs->num_corr == 0) return CB_OK;
    ++gn->steps;
    gn->cg_total += hs->cg_iters;
    gn->cg_last = hs->cg_iters;
    gn->cg_err = hs->cg_err;
    float mx;
    std::memcpy(&mx, &hs->max_delta_bits, sizeof(float));
    if (mx < tol2) {
      gn->converged = 1;
      break;
    }
  }
  return CB_OK;
}

// The estimator's output over the m blocks (:701-712, :1832-1843; compose: preApply with projection, else the plain
// transforms) and the max of |dR_j - I|_F^2 + |dt_j|^2. warp_next (one block per point only): also the warped points
// for the next search and, into *num_corr, the correspondences of the last search.
int apply_update(WarpCore* w, bool compose, bool warp_next, float* last_delta_sq, uint32_t* num_corr) {
  cb_context* ctx = w->ctx;
  CB_CUDA(cudaMemsetAsync(w->d_stats, 0, sizeof(WarpStats), ctx->stream));
  if (w->m) {
    warp_compose_kernel<<<grid_for(ctx, w->m), kBlock, 0, ctx->stream>>>(
        w->m, w->src->d_raw, w->d_xs, w->d_T, compose, warp_next ? w->d_warped : nullptr,
        warp_next ? w->d_nn : nullptr, w->d_stats);
    ctx->launches += 1;
    CB_CUDA(cudaGetLastError());
  }
  CB_CUDA(cudaMemcpyAsync(w->h_stats, w->d_stats, sizeof(WarpStats), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  std::memcpy(last_delta_sq, &w->h_stats->last_delta_bits, sizeof(float));
  if (num_corr) *num_corr = w->h_stats->num_corr;
  return CB_OK;
}

}  // namespace
