// Per-correspondence accumulation of the ICP estimators (product code, sm_90a), shared by the fused
// search+accumulate kernel (icp_kernels.cu) and the pair-list kernel of the non-default correspondence
// engine modes (icp_engine.cu).
//   kModeP2P      Kabsch moments  n, sum d, sum q, sum d q^T          transform_estimation.hpp:25-34
//   kModeCombined Gauss-Newton normal equations (point-to-point + point-to-plane / symmetric terms)
//                                                                      transform_estimation.hpp:298-343, :669-715
#pragma once
#include "icp_kernels.cuh"

namespace cb {

__device__ __forceinline__ constexpr int ut(int r, int c) { return r * 6 - (r * (r - 1)) / 2 + (c - r); }

// dp = matched destination point, (qx,qy,qz) = T * source point. load_dst_normal() / load_src_normal()
// are only invoked when the metric needs them (has_pl / have_src_normal).
// Args: anything with the fields T, Tin (Rigid), dm, sm (float[3]), w_pt, w_pl, wk_pt, wk_pl, wc_pt, wc_pl — IcpArgs,
// or the loop kernel's per-block context. corr_d2 = the correspondence's value (squared distance found by the search of
// this ICP iteration): input of the RBF correspondence weight evaluators (common_pair_evaluators.hpp:46-79). kIdentityTin = true skips the (identity) inner Gauss-Newton transform of the first pass:
// (1*x + (0*y + 0*z)) + 0 == x bit for bit for finite x.
template <int MODE, bool kIdentityTin = false, class Args, class LoadDstNormal, class LoadSrcNormal>
__device__ __forceinline__ void accumulate_pair(double* acc, const Args& a, bool has_pt, bool has_pl,
                                                const float4 dp, float qx, float qy, float qz, bool have_src_normal,
                                                LoadDstNormal load_dst_normal, LoadSrcNormal load_src_normal,
                                                float corr_d2 = 0.f) {
  if constexpr (MODE == kModeP2P) {
    const double dx = dp.x, dy = dp.y, dz = dp.z, x = qx, y = qy, z = qz;
    acc[0] += 1.0;
    acc[1] += dx; acc[2] += dy; acc[3] += dz;
    acc[4] += x;  acc[5] += y;  acc[6] += z;
    acc[7] += dx * x;  acc[8] += dx * y;  acc[9] += dx * z;
    acc[10] += dy * x; acc[11] += dy * y; acc[12] += dy * z;
    acc[13] += dz * x; acc[14] += dz * y; acc[15] += dz * z;
  } else if constexpr (MODE == kModeP2PCentered) {
    // the same 16 moments about the pivots dm (dst mean) and sm (T * src mean): no cancellation in
    // sigma = (sum d' q'^T)/n - mu_d' mu_q'^T for clouds far from the origin (solve_core.hpp)
    const double dx = (double)dp.x - (double)a.dm[0], dy = (double)dp.y - (double)a.dm[1], dz = (double)dp.z - (double)a.dm[2];
    const double x = (double)qx - (double)a.sm[0], y = (double)qy - (double)a.sm[1], z = (double)qz - (double)a.sm[2];
    acc[0] += 1.0;
    acc[1] += dx; acc[2] += dy; acc[3] += dz;
    acc[4] += x;  acc[5] += y;  acc[6] += z;
    acc[7] += dx * x;  acc[8] += dx * y;  acc[9] += dx * z;
    acc[10] += dy * x; acc[11] += dy * y; acc[12] += dy * z;
    acc[13] += dz * x; acc[14] += dz * y; acc[15] += dz * z;
  } else if constexpr (MODE == kModeCombined) {
    // d = dst - dst_mean ; s = Tin * (q - T*src_mean)           transform_estimation.hpp:300,304
    const float d0 = __fsub_rn(dp.x, a.dm[0]), d1 = __fsub_rn(dp.y, a.dm[1]), d2 = __fsub_rn(dp.z, a.dm[2]);
    float s0, s1, s2;
    if constexpr (kIdentityTin) {
      s0 = __fsub_rn(qx, a.sm[0]);
      s1 = __fsub_rn(qy, a.sm[1]);
      s2 = __fsub_rn(qz, a.sm[2]);
    } else {
      rule::transform_point(a.Tin, __fsub_rn(qx, a.sm[0]), __fsub_rn(qy, a.sm[1]), __fsub_rn(qz, a.sm[2]), s0, s1, s2);
    }
    const float v0 = __fadd_rn(d0, s0), v1 = __fadd_rn(d1, s1), v2 = __fadd_rn(d2, s2);
    const float e0 = __fsub_rn(d0, s0), e1 = __fsub_rn(d1, s1), e2 = __fsub_rn(d2, s2);
    acc[0] += 1.0;
    double* A = acc + 1;
    double* b = acc + 22;
    if (has_pt) {
      // eq_vecs E = [ [v]x ; I ] (6x3, :306-316)  ->  E E^T = [ |v|^2 I - v v^T , [v]x ; -[v]x , I ],
      // E e = [ v x e ; e ]
      // weight = point_to_point_weight * point_corr_evaluator(i, j, value), in float      transform_estimation.hpp:302-304
      const double w = a.wk_pt ? (double)__fmul_rn(a.w_pt, expf(__fmul_rn(a.wc_pt, corr_d2))) : (double)a.w_pt;
      const double V0 = v0, V1 = v1, V2 = v2, E0 = e0, E1 = e1, E2 = e2;
      A[ut(0, 0)] += w * (V1 * V1 + V2 * V2);
      A[ut(0, 1)] -= w * (V0 * V1);
      A[ut(0, 2)] -= w * (V0 * V2);
      A[ut(1, 1)] += w * (V0 * V0 + V2 * V2);
      A[ut(1, 2)] -= w * (V1 * V2);
      A[ut(2, 2)] += w * (V0 * V0 + V1 * V1);
      A[ut(0, 4)] -= w * V2;
      A[ut(0, 5)] += w * V1;
      A[ut(1, 3)] += w * V2;
      A[ut(1, 5)] -= w * V0;
      A[ut(2, 3)] -= w * V1;
      A[ut(2, 4)] += w * V0;
      A[ut(3, 3)] += w;
      A[ut(4, 4)] += w;
      A[ut(5, 5)] += w;
      b[0] += w * (V1 * E2 - V2 * E1);
      b[1] += w * (V2 * E0 - V0 * E2);
      b[2] += w * (V0 * E1 - V1 * E0);
      b[3] += w * E0;
      b[4] += w * E1;
      b[5] += w * E2;
    }
    if (has_pl) {
      const float4 np = load_dst_normal();
      float n0 = np.x, n1 = np.y, n2 = np.z;
      if (have_src_normal) {  // symmetric metric: n = n_dst + R_in (R_T n_src)        :705-706
        const float4 sn = load_src_normal();
        float r0, r1, r2, t0, t1, t2;
        rotate_rigid(a.T, sn.x, sn.y, sn.z, r0, r1, r2);
        if constexpr (kIdentityTin) {
          t0 = r0;
          t1 = r1;
          t2 = r2;
        } else {
          rotate_rigid(a.Tin, r0, r1, r2, t0, t1, t2);
        }
        n0 = __fadd_rn(n0, t0);
        n1 = __fadd_rn(n1, t1);
        n2 = __fadd_rn(n2, t2);
      }
      // a = [ (d + s) x n ; n ],  r = n . (d - s)                                  :337-341
      const float c0 = __fsub_rn(__fmul_rn(v1, n2), __fmul_rn(v2, n1));
      const float c1 = __fsub_rn(__fmul_rn(v2, n0), __fmul_rn(v0, n2));
      const float c2 = __fsub_rn(__fmul_rn(v0, n1), __fmul_rn(v1, n0));
      const double av[6] = {c0, c1, c2, n0, n1, n2};
      const double rd = (double)n0 * e0 + ((double)n1 * e1 + (double)n2 * e2);
      const double w = a.wk_pl ? (double)__fmul_rn(a.w_pl, expf(__fmul_rn(a.wc_pl, corr_d2))) : (double)a.w_pl;  // :331-333
#pragma unroll
      for (int r = 0; r < 6; r++) {
        const double wr = w * av[r];
#pragma unroll
        for (int c = r; c < 6; c++) A[ut(r, c)] += wr * av[c];
        b[r] += wr * rd;
      }
    }
  }
}

}  // namespace cb
