// Pinned rule of the robust (minimum-covariance-determinant) normal estimation (robust_normals.cu), shared by the
// host and the device. MinimumCovarianceDeterminant (core/covariance.hpp:185-371) cannot be reproduced bit for bit:
// it seeds a fresh std::random_device per point, orders the kept subset with std::partial_sort and leaves the 3x3
// inverse and determinant to Eigen. This header fixes one rule for each of those, and holds the fp32 arithmetic the
// kernel and the oracle (oracle/robust_normals_oracle.cpp) both run; DESIGN §4.15 states the contract.
//
//   * Randomness: every point runs its own std::minstd_rand0 (libstdc++'s std::default_random_engine), seeded with
//     point_seed(seed, original index). Each draw is std::uniform_int_distribution<size_t>(0, size - 1) as
//     libstdc++ implements it for this engine (the two-division downscale with rejection). Draws index the
//     neighbourhood in search order (ascending (d2, index)).
//   * Selection of the h kept points: ascending (Mahalanobis key, neighbour position); NaN keys sort as +inf,
//     -0 as +0. Keys map to order-preserving unsigned integers, so a negative key (indefinite sample covariance)
//     sorts below zero.
//   * 3x3 algebra: cofactors, determinant, inverse and the quadratic form below, one rounding per operation.
// tests/cpp/test_mcd_rule.cpp compiles this header for the host (-ffp-contract=off) and checks the generator and
// the draws against the installed libstdc++, the key order, and the inverse and determinant against float64.
#pragma once
#include <cstdint>
#include <cstring>
#include <cmath>

#if defined(__CUDACC__)
#define CB_MCD_HD __host__ __device__ __forceinline__
#else
#define CB_MCD_HD inline
#endif

namespace cb {
namespace mcd {

constexpr int kMaxK = 128;          // neighbourhood size the kernel stages per warp
constexpr int kMaxMinSample = 32;   // largest minimum sample size (one draw per lane)

// per-point status
enum : uint8_t { kOk = 0, kTooFew = 1, kRejected = 2, kNoFiniteTrial = 3 };

// ---- fp32 with one rounding per operation ------------------------------------------------------------------
CB_MCD_HD float add(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
CB_MCD_HD float sub(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
CB_MCD_HD float mul(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
CB_MCD_HD float div(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}
CB_MCD_HD uint32_t float_bits(float f) {
#if defined(__CUDA_ARCH__)
  return __float_as_uint(f);
#else
  uint32_t b;
  std::memcpy(&b, &f, 4);
  return b;
#endif
}

// ---- randomness ------------------------------------------------------------------------------------------
// MurmurHash3's 32-bit finaliser: full avalanche, so neighbouring indices give unrelated minstd seeds (minstd's
// first outputs from seeds s and s + 1 differ by exactly 16807).
CB_MCD_HD uint32_t fmix32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x85ebca6bu;
  x ^= x >> 13;
  x *= 0xc2b2ae35u;
  x ^= x >> 16;
  return x;
}
CB_MCD_HD uint32_t point_seed(uint32_t seed, uint32_t index) { return fmix32(seed ^ fmix32(index + 0x9e3779b9u)); }

// std::minstd_rand0(s): x = s mod (2^31 - 1), 0 -> 1; next: x = 16807 x mod (2^31 - 1), returned.
CB_MCD_HD uint32_t minstd_seed(uint32_t s) {
  const uint32_t x = s % 2147483647u;
  return x == 0u ? 1u : x;
}
CB_MCD_HD uint32_t minstd_next(uint32_t& x) {
  x = (uint32_t)(((uint64_t)x * 16807u) % 2147483647u);
  return x;
}

// std::uniform_int_distribution<size_t>(0, n - 1)(minstd), n >= 1: the engine's range (max - min = 2^31 - 3) is
// wider than n - 1, so libstdc++ downscales: scaling = range / n, past = n * scaling, draw (x - 1) until it is
// below past, return it / scaling. The expected number of draws is below 1 + n / 2^31.
CB_MCD_HD uint32_t uniform_below(uint32_t& x, uint32_t n) {
  const uint32_t scaling = 2147483645u / n;
  const uint32_t past = n * scaling;
  uint32_t r;
  do {
    r = minstd_next(x) - 1u;
  } while (r >= past);
  return r / scaling;
}

// ---- subset size --------------------------------------------------------------------------------------------
// h = min(max(min_size, llround(ratio * size)), size) with ratio * size in fp32. A negative llround converts to a
// huge size_t in the reference, so it gives h = size; so does a product above size (+inf included).
CB_MCD_HD uint32_t subset_size(float ratio, uint32_t size, uint32_t min_size) {
  const float r = roundf(mul(ratio, (float)size));  // halfway away from zero, like llround
  if (!(r >= 0.f)) return size;
  const uint32_t h = r >= (float)size ? size : (uint32_t)r;
  return h < min_size ? min_size : h;
}

// ---- selection order ---------------------------------------------------------------------------------------
CB_MCD_HD uint32_t key_bits(float f) {
  if (f != f) f = INFINITY;
  if (f == 0.f) f = 0.f;  // -0 -> +0
  const uint32_t b = float_bits(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
// (key, position) as one unsigned integer: ascending order = the selection order
CB_MCD_HD uint64_t sort_key(float key, uint32_t pos) { return ((uint64_t)key_bits(key) << 32) | pos; }

// ---- 3x3 symmetric algebra (a = xx, xy, xz, yy, yz, zz) ----------------------------------------------------
CB_MCD_HD void cofactors(const float (&a)[6], float (&c)[6]) {
  c[0] = sub(mul(a[3], a[5]), mul(a[4], a[4]));
  c[1] = sub(mul(a[2], a[4]), mul(a[1], a[5]));
  c[2] = sub(mul(a[1], a[4]), mul(a[2], a[3]));
  c[3] = sub(mul(a[0], a[5]), mul(a[2], a[2]));
  c[4] = sub(mul(a[1], a[2]), mul(a[0], a[4]));
  c[5] = sub(mul(a[0], a[3]), mul(a[1], a[1]));
}
// Laplace expansion along the first row: (a00 c00 + a01 c01) + a02 c02
CB_MCD_HD float det_from(const float (&a)[6], const float (&c)[6]) {
  return add(add(mul(a[0], c[0]), mul(a[1], c[1])), mul(a[2], c[2]));
}
CB_MCD_HD float determinant(const float (&a)[6]) {
  float c[6];
  cofactors(a, c);
  return det_from(a, c);
}
// inverse = cofactors * (1 / det); a singular matrix gives Inf / NaN entries (and keys), never a fault
CB_MCD_HD void inverse(const float (&a)[6], float (&m)[6]) {
  float c[6];
  cofactors(a, c);
  const float r = div(1.f, det_from(a, c));
#pragma unroll
  for (int i = 0; i < 6; i++) m[i] = mul(c[i], r);
}
// d^T M d = (dx r0 + dy r1) + dz r2, each row r_i = (m_i0 dx + m_i1 dy) + m_i2 dz
CB_MCD_HD float mahalanobis2(const float (&m)[6], float dx, float dy, float dz) {
  const float r0 = add(add(mul(m[0], dx), mul(m[1], dy)), mul(m[2], dz));
  const float r1 = add(add(mul(m[1], dx), mul(m[3], dy)), mul(m[4], dz));
  const float r2 = add(add(mul(m[2], dx), mul(m[4], dy)), mul(m[5], dz));
  return add(add(mul(dx, r0), mul(dy, r1)), mul(dz, r2));
}

// ---- mean and covariance -----------------------------------------------------------------------------------
// Covariance::operator() (core/covariance.hpp:121-135) over count >= 2 points taken in order: serial sums,
// mean = (1 / count) * sum, cov = (1 / (count - 1)) * sum of outer products. get(j, x, y, z) loads point j. The
// same arithmetic as normals_knn_kernel, so a subset equal to the whole neighbourhood gives its covariance bits.
template <class Get>
CB_MCD_HD void mean_cov(uint32_t count, Get get, float (&mean)[3], float (&cv)[6]) {
  float mx = 0.f, my = 0.f, mz = 0.f;
  for (uint32_t j = 0; j < count; j++) {
    float x, y, z;
    get(j, x, y, z);
    mx = add(mx, x);
    my = add(my, y);
    mz = add(mz, z);
  }
  const float inv = div(1.0f, (float)count);
  mean[0] = mul(inv, mx);
  mean[1] = mul(inv, my);
  mean[2] = mul(inv, mz);
#pragma unroll
  for (int c = 0; c < 6; c++) cv[c] = 0.f;
  for (uint32_t j = 0; j < count; j++) {
    float x, y, z;
    get(j, x, y, z);
    const float dx = sub(x, mean[0]), dy = sub(y, mean[1]), dz = sub(z, mean[2]);
    cv[0] = add(cv[0], mul(dx, dx));
    cv[1] = add(cv[1], mul(dx, dy));
    cv[2] = add(cv[2], mul(dx, dz));
    cv[3] = add(cv[3], mul(dy, dy));
    cv[4] = add(cv[4], mul(dy, dz));
    cv[5] = add(cv[5], mul(dz, dz));
  }
  const float invm1 = div(1.0f, (float)(count - 1));
#pragma unroll
  for (int c = 0; c < 6; c++) cv[c] = mul(invm1, cv[c]);
}

// A trial counts only with a finite determinant below the best so far (which starts at FLT_MAX).
CB_MCD_HD bool improves(float det, float best) { return det - det == 0.f && det < best; }

}  // namespace mcd
}  // namespace cb
