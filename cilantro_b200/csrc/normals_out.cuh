// The last step of every normal estimation (normals.cu, robust_normals.cu): the eigen solve of the neighbourhood
// covariance, the orientation step, and the stores into the cloud and the optional outputs.
#pragma once
#include <cmath>

#include "cb_internal.hpp"
#include "sym3_eigen.cuh"

namespace cb {

struct NormalOut {
  float* raw_nrm;    // 3n, original order
  float4* nrm;       // n, cell-sorted
  float* curvature;  // n, original order, or nullptr
  float* cov6;       // 6n, original order, or nullptr
  float vx, vy, vz;  // view point
  int use_vp;
  int use_ref;  // orient by the cloud's current normals (takes precedence over the view point)
};

__device__ __forceinline__ void finish_point(const NormalOut& o, uint32_t qi, int oi, float px, float py, float pz,
                                             bool valid, const float (&cv)[6]) {
  const float nan = __int_as_float(0x7fc00000);
  float w[3], nv[3] = {nan, nan, nan}, curv = nan;
  if (valid) {
    sym3_smallest(cv, w, nv, curv);
    if (o.use_ref) {
      // eigenvectors().col(0).dot(ref_normals.col(i)) < 0 -> flip (normal_estimation.hpp:351-355)
      const float4 r = o.nrm[qi];
      const float d = __fadd_rn(__fmul_rn(nv[0], r.x), __fadd_rn(__fmul_rn(nv[1], r.y), __fmul_rn(nv[2], r.z)));
      if (d < 0.f) {
        nv[0] = -nv[0];
        nv[1] = -nv[1];
        nv[2] = -nv[2];
      }
    } else if (o.use_vp) {
      // eigenvectors().col(0).dot(view_point - p) < 0 -> flip (normal_estimation.hpp:325-329)
      const float ex = __fsub_rn(o.vx, px), ey = __fsub_rn(o.vy, py), ez = __fsub_rn(o.vz, pz);
      const float d = __fadd_rn(__fmul_rn(nv[0], ex), __fadd_rn(__fmul_rn(nv[1], ey), __fmul_rn(nv[2], ez)));
      if (d < 0.f) {
        nv[0] = -nv[0];
        nv[1] = -nv[1];
        nv[2] = -nv[2];
      }
    }
  }
  o.nrm[qi] = make_float4(nv[0], nv[1], nv[2], 0.f);
  o.raw_nrm[3 * (size_t)oi] = nv[0];
  o.raw_nrm[3 * (size_t)oi + 1] = nv[1];
  o.raw_nrm[3 * (size_t)oi + 2] = nv[2];
  if (o.curvature) o.curvature[oi] = curv;  // :389
  if (o.cov6) {
#pragma unroll
    for (int c = 0; c < 6; c++) o.cov6[6 * (size_t)oi + c] = valid ? cv[c] : nan;
  }
}

// The orientation inputs of cb_cloud_estimate_normals{,_mcd}: the view point when it is finite
// (view_point_.allFinite(), normal_estimation.hpp:283) and the cloud's current normals when asked for and present.
inline void set_orientation(NormalOut& o, const float* view_point3, bool use_ref) {
  o.use_vp = view_point3 && std::isfinite(view_point3[0]) && std::isfinite(view_point3[1]) &&
             std::isfinite(view_point3[2]);
  o.use_ref = use_ref ? 1 : 0;
  o.vx = o.use_vp ? view_point3[0] : 0.f;
  o.vy = o.use_vp ? view_point3[1] : 0.f;
  o.vz = o.use_vp ? view_point3[2] : 0.f;
}

}  // namespace cb
