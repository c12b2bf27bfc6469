// The exclusion-cache rule of the device-resident ICP loop (icp_loop.cu), as ONE function that compiles for the device
// (the cached-pass kernel calls it) and for the host (tests/cpp/test_cache_rule.cpp drives it against a brute-force
// search with the tightest exclusion radius there is: the computed distance of the second-nearest point).
//
// The claim it implements. A search under transform T_k returned for source point s the nearest reference point m and a
// radius r such that every OTHER reference point is at least r away from q_k = T_k s. Under T_{k+1} the query sits at
// q = T_{k+1} s, |q - q_k| <= dl, so every other point is at least r2 = r - dl away from q (triangle inequality). If the
// match's distance under T_{k+1}, evaluated with the contract arithmetic (the very number a search would compute for it),
// satisfies d2 < lim = r2^2 (1 - 2^-17), the match is still the unique nearest neighbour and (m, d2) is what a full
// search returns, bit for bit. dl is rounded up (+2^-18), r2 and lim are rounded down: the margins are far above the
// few-ulp error of the fp32 distance evaluation, and an exact tie can never pass the strict test. The same bound decides
// "nothing is inside the correspondence radius": max_d2 <= lim.
//
// No CUDA headers: the host build needs <cfenv> / <cmath> only and must be compiled with -frounding-math
// -ffp-contract=off (directed rounding through the floating-point environment).
#pragma once
#if defined(__CUDACC__)
#define CB_RULE_HD __host__ __device__ __forceinline__
#else
#define CB_RULE_HD inline
#endif
#if !defined(__CUDA_ARCH__)
#include <cfenv>
#include <cmath>
#endif

namespace cb {
namespace rule {

constexpr float kUp18 = 1.0000038146972656f;    // 1 + 2^-18
constexpr float kDown18 = 0.9999961853027344f;  // 1 - 2^-18
constexpr float kDown17 = 0.9999923706054688f;  // 1 - 2^-17

#if defined(__CUDA_ARCH__)
CB_RULE_HD float add_rn(float a, float b) { return __fadd_rn(a, b); }
CB_RULE_HD float sub_rn(float a, float b) { return __fsub_rn(a, b); }
CB_RULE_HD float mul_rn(float a, float b) { return __fmul_rn(a, b); }
CB_RULE_HD float mul_ru(float a, float b) { return __fmul_ru(a, b); }
CB_RULE_HD float mul_rd(float a, float b) { return __fmul_rd(a, b); }
CB_RULE_HD float sub_rd(float a, float b) { return __fsub_rd(a, b); }
CB_RULE_HD float fma_ru(float a, float b, float c) { return __fmaf_ru(a, b, c); }
CB_RULE_HD float sqrt_ru(float a) { return __fsqrt_ru(a); }
CB_RULE_HD float sqrt_rd(float a) { return __fsqrt_rd(a); }
#else
// host twins: IEEE operations under the requested rounding direction (volatile operands: no folding, no reordering)
template <class F>
inline float directed(int mode, F f) {
  const int old = std::fegetround();
  std::fesetround(mode);
  volatile float r = f();
  std::fesetround(old);
  return r;
}
inline float add_rn(float a, float b) { volatile float x = a, y = b; volatile float r = x + y; return r; }
inline float sub_rn(float a, float b) { volatile float x = a, y = b; volatile float r = x - y; return r; }
inline float mul_rn(float a, float b) { volatile float x = a, y = b; volatile float r = x * y; return r; }
inline float mul_ru(float a, float b) { volatile float x = a, y = b; return directed(FE_UPWARD, [&] { return x * y; }); }
inline float mul_rd(float a, float b) { volatile float x = a, y = b; return directed(FE_DOWNWARD, [&] { return x * y; }); }
inline float sub_rd(float a, float b) { volatile float x = a, y = b; return directed(FE_DOWNWARD, [&] { return x - y; }); }
inline float fma_ru(float a, float b, float c) {
  volatile float x = a, y = b, z = c;
  return directed(FE_UPWARD, [&] { return std::fmaf(x, y, z); });
}
inline float sqrt_ru(float a) { volatile float x = a; return directed(FE_UPWARD, [&] { return std::sqrt((float)x); }); }
inline float sqrt_rd(float a) { volatile float x = a; return directed(FE_DOWNWARD, [&] { return std::sqrt((float)x); }); }
#endif

// q = R s + t with the contract arithmetic: q_r = (R_r0 x + (R_r1 y + R_r2 z)) + t_r: the transform every search kernel
// applies to its queries
template <class RigidT>
CB_RULE_HD void transform_point(const RigidT& T, float x, float y, float z, float& qx, float& qy, float& qz) {
  qx = add_rn(add_rn(mul_rn(T.r[0], x), add_rn(mul_rn(T.r[1], y), mul_rn(T.r[2], z))), T.t[0]);
  qy = add_rn(add_rn(mul_rn(T.r[3], x), add_rn(mul_rn(T.r[4], y), mul_rn(T.r[5], z))), T.t[1]);
  qz = add_rn(add_rn(mul_rn(T.r[6], x), add_rn(mul_rn(T.r[7], y), mul_rn(T.r[8], z))), T.t[2]);
}

// d2 = ((dx dx) + dy dy) + dz dz, d = q - p: the distance every search kernel computes
CB_RULE_HD float contract_d2(float qx, float qy, float qz, float px, float py, float pz) {
  const float dx = sub_rn(qx, px), dy = sub_rn(qy, py), dz = sub_rn(qz, pz);
  float d2 = mul_rn(dx, dx);
  d2 = add_rn(d2, mul_rn(dy, dy));
  d2 = add_rn(d2, mul_rn(dz, dz));
  return d2;
}

// what a search stores for its query: the radius inside which only the match lives (D2 = the search's lower bound of
// every other point's squared distance; 0 = unknown -> nothing cached)
CB_RULE_HD float cache_radius(float D2) { return (D2 > 0.f) ? mul_rd(sqrt_rd(D2), kDown18) : 0.f; }

struct Verdict {
  bool miss;         // true: the query has to be searched again
  bool pair;         // !miss and the cached match is the correspondence (inside the radius); its squared distance is d2
  float r2;          // the radius to store back when !miss (the bound shrinks by the motion of every iteration)
  float d2;
  float qx, qy, qz;  // T s
};

// T / Tp: this iteration's and the previous iteration's transform; (sx, sy, sz): the source point; rc > 0: its cached
// radius; seed: position of its cached match (-1 = nothing was inside the correspondence radius); load_match():
// coordinates of that match (called only when seed >= 0); p receives them.
template <class RigidT, class PointT, class LoadMatch>
CB_RULE_HD void cached_match_test(const RigidT& T, const RigidT& Tp, float sx, float sy, float sz, float rc, int seed,
                                  float max_d2, LoadMatch&& load_match, PointT& p, Verdict& v) {
  v.miss = true;
  v.pair = false;
  v.r2 = 0.f;
  v.d2 = 0.f;
  float ox, oy, oz;
  transform_point(T, sx, sy, sz, v.qx, v.qy, v.qz);
  transform_point(Tp, sx, sy, sz, ox, oy, oz);
  const float ex = sub_rn(v.qx, ox), ey = sub_rn(v.qy, oy), ez = sub_rn(v.qz, oz);
  // upper bound of the distance the query moved since the previous iteration
  const float dl = mul_ru(sqrt_ru(fma_ru(ez, ez, fma_ru(ey, ey, mul_ru(ex, ex)))), kUp18);
  const float r2 = sub_rd(rc, dl);
  if (r2 > 0.f) {
    // every reference point other than the match has a computed d2 above lim under the current transform
    const float lim = mul_rd(mul_rd(r2, r2), kDown17);
    if (seed >= 0) {
      p = load_match();
      v.d2 = contract_d2(v.qx, v.qy, v.qz, p.x, p.y, p.z);
      if (v.d2 < max_d2) {
        if (v.d2 < lim) {  // still the unique nearest neighbour, inside the radius
          v.miss = false;
          v.pair = true;
        }
      } else if (max_d2 <= lim) {  // the match left the radius and nothing else is inside it
        v.miss = false;
      }
    } else if (max_d2 <= lim) {  // nothing was within the radius and nothing can have entered it
      v.miss = false;
    }
    v.r2 = r2;
  }
}

}  // namespace rule
}  // namespace cb
