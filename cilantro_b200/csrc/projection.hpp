// Which pixel a point lands in (DESIGN §4.20, §4.21): ONE function, compiled for the device (the z-buffer of
// depth_images.cu and the projective correspondence search of projective_search.cu / icp_loop.cu) and for the host.
//   c = E^-1 p with the isometry inverse L = R^T, tr = -(L t) (Eigen's dot order (a0 b0 + a1 b1) + a2 b2)
//   skipped unless c.z > 0
//   x = llround(inv_z * dot(K row 0, c)), y likewise from row 1 (half away from zero); skipped when non-finite or
//   outside [0, w) x [0, h): a projection in (-0.5, 0) lands on pixel 0
#pragma once
#include <cstdint>
#include "cache_rule.hpp"

namespace cb {

struct Projection {
  float K0[3], K1[3];  // rows 0 and 1 of the intrinsics
  int extr;            // camera frame = L p + tr (extrinsics.inverse()); 0: p itself
  float L[9], tr[3];
  uint32_t w, h;
};

// A projective correspondence search attached to an ICP object (cb_icp_set_projection, cb_warp_icp_set_projection,
// cb_sparse_warp_icp_set_projection; built by build_projective_map in projective_search.cu, DESIGN §4.21, §4.22).
struct ProjectiveMap {
  bool on = false;
  Projection prj;
  int* d_map = nullptr;  // w * h: sorted position of the destination point each pixel shows, -1 empty (owned by the
                         // object)
};

namespace rule {
#if defined(__CUDA_ARCH__)
CB_RULE_HD float div_rn(float a, float b) { return __fdiv_rn(a, b); }
CB_RULE_HD float round_away(float a) { return roundf(a); }
CB_RULE_HD bool finite(float a) { return isfinite(a); }
#else
inline float div_rn(float a, float b) { volatile float x = a, y = b; volatile float r = x / y; return r; }
inline float round_away(float a) { return std::round(a); }
inline bool finite(float a) { return std::isfinite(a); }
#endif
CB_RULE_HD float dot3(const float* a, float b0, float b1, float b2) {
  return add_rn(add_rn(mul_rn(a[0], b0), mul_rn(a[1], b1)), mul_rn(a[2], b2));
}
}  // namespace rule

// K: row-major 3 x 3; E: row-major 3 x 4 [R | t] or nullptr (identity)
inline Projection make_projection(const float* K, const float* E, uint32_t w, uint32_t h) {
  Projection P{};
  for (int j = 0; j < 3; j++) {
    P.K0[j] = K[j];
    P.K1[j] = K[3 + j];
  }
  P.w = w;
  P.h = h;
  if (E) {
    P.extr = 1;
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) P.L[3 * i + j] = E[4 * j + i];
    for (int i = 0; i < 3; i++) P.tr[i] = -rule::dot3(P.L + 3 * i, E[3], E[7], E[11]);
  }
  return P;
}

// true: (x, y, z) lands on pixel (px, py) at camera-frame depth cz
CB_RULE_HD bool project_pixel(const Projection& P, float x, float y, float z, uint32_t& px, uint32_t& py, float& cz) {
  if (P.extr) {
    const float c0 = rule::add_rn(rule::dot3(P.L, x, y, z), P.tr[0]);
    const float c1 = rule::add_rn(rule::dot3(P.L + 3, x, y, z), P.tr[1]);
    const float c2 = rule::add_rn(rule::dot3(P.L + 6, x, y, z), P.tr[2]);
    x = c0;
    y = c1;
    z = c2;
  }
  if (!(z > 0.0f)) return false;  // z <= 0; a NaN z projects to NaN and is skipped below in any case
  const float inv_z = rule::div_rn(1.0f, z);
  const float fx = rule::mul_rn(inv_z, rule::dot3(P.K0, x, y, z)), fy = rule::mul_rn(inv_z, rule::dot3(P.K1, x, y, z));
  if (!rule::finite(fx) || !rule::finite(fy)) return false;
  const float rx = rule::round_away(fx), ry = rule::round_away(fy);  // llround: half away from zero
  if (!(rx >= 0.0f && ry >= 0.0f) || (double)rx >= (double)P.w || (double)ry >= (double)P.h) return false;
  px = (uint32_t)rx;
  py = (uint32_t)ry;
  cz = z;
  return true;
}

}  // namespace cb
