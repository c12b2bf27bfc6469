// Smallest eigenpair of a symmetric 3x3 in fp32 registers (product code, sm_90a): the eigen solve of the normal
// estimation (normals.cu), in a header of its own so that tests/cuda/solve_harness.cu runs the shipped code.
#pragma once

namespace cb {

// Cyclic Jacobi on a symmetric 3x3 (a = xx,xy,xz,yy,yz,zz). Eigenvalues ascending in w, v0 = unit
// eigenvector of w[0]. The matrix is scaled by its largest |entry| first, like
// SelfAdjointEigenSolver::compute, so tiny covariances (metric clouds in mm^2 .. m^2) keep their
// relative accuracy.
__device__ __forceinline__ void jacobi_rotate(float& app, float& aqq, float& apq, float& arp, float& arq, float& v0p,
                                              float& v0q, float& v1p, float& v1q, float& v2p, float& v2q) {
  if (fabsf(apq) < 1e-30f) return;
  const float theta = (aqq - app) / (2.f * apq);
  const float t = copysignf(1.f, theta) / (fabsf(theta) + sqrtf(theta * theta + 1.f));
  const float c = rsqrtf(t * t + 1.f);
  const float s = t * c;
  app -= t * apq;
  aqq += t * apq;
  apq = 0.f;
  const float rp = c * arp - s * arq, rq = s * arp + c * arq;
  arp = rp;
  arq = rq;
  float a, b;
  a = c * v0p - s * v0q; b = s * v0p + c * v0q; v0p = a; v0q = b;
  a = c * v1p - s * v1q; b = s * v1p + c * v1q; v1p = a; v1q = b;
  a = c * v2p - s * v2q; b = s * v2p + c * v2q; v2p = a; v2q = b;
}

// The smallest eigenpair and the curvature w0 / (w0 + w1 + w2) (normal_estimation.hpp:389) of cv.
// Below a largest |entry| of 2^-126 every entry is subnormal or zero: 1 / scale overflows to +inf below 2^-128, and
// the eigenvalues would be subnormal. Such a matrix is multiplied by 2^64 first (exact), solved as any other, and
// only its eigenvalues are multiplied back by 2^-64. The curvature is taken before that step, so it keeps all its
// bits: an exact power-of-two scaling of a normal-range matrix gets that matrix's normal and curvature bit for bit.
// A NaN or infinite entry makes every output NaN (an infinite entry: as Eigen's solver, which divides by the
// infinite scale); the zero matrix gives n = e_x, w = 0 and curv = NaN (0 / 0).
__device__ __forceinline__ void sym3_smallest(const float (&cv)[6], float (&w)[3], float (&n)[3], float& curv) {
  bool finite = true;
#pragma unroll
  for (int c = 0; c < 6; c++) finite = finite && fabsf(cv[c]) <= 3.402823466e38f;
  if (!finite) {
    w[0] = w[1] = w[2] = n[0] = n[1] = n[2] = curv = __int_as_float(0x7fc00000);
    return;
  }
  float scale = fmaxf(fmaxf(fabsf(cv[0]), fabsf(cv[1])), fmaxf(fabsf(cv[2]), fabsf(cv[3])));
  scale = fmaxf(scale, fmaxf(fabsf(cv[4]), fabsf(cv[5])));
  if (!(scale > 0.f)) {  // zero matrix: eigenvectors = identity
    w[0] = w[1] = w[2] = scale;
    n[0] = 1.f;
    n[1] = 0.f;
    n[2] = 0.f;
    curv = w[0] / (w[0] + w[1] + w[2]);
    return;
  }
  const bool tiny = scale < 0x1p-126f;
  const float up = tiny ? 0x1p64f : 1.f;
  scale *= up;
  const float inv = 1.f / scale;
  float a00 = cv[0] * up * inv, a01 = cv[1] * up * inv, a02 = cv[2] * up * inv, a11 = cv[3] * up * inv,
        a12 = cv[4] * up * inv, a22 = cv[5] * up * inv;
  float v00 = 1.f, v01 = 0.f, v02 = 0.f, v10 = 0.f, v11 = 1.f, v12 = 0.f, v20 = 0.f, v21 = 0.f, v22 = 1.f;
#pragma unroll 1
  for (int sweep = 0; sweep < 8; ++sweep) {
    const float off = fabsf(a01) + fabsf(a02) + fabsf(a12);
    if (off < 1e-12f) break;
    jacobi_rotate(a00, a11, a01, a02, a12, v00, v01, v10, v11, v20, v21);  // (p,q,r) = (0,1,2)
    jacobi_rotate(a00, a22, a02, a01, a12, v00, v02, v10, v12, v20, v22);  // (0,2,1)
    jacobi_rotate(a11, a22, a12, a01, a02, v01, v02, v11, v12, v21, v22);  // (1,2,0)
  }
  // ascending eigenvalues; n = column of the smallest
  float l0 = a00, l1 = a11, l2 = a22;
  float nx = v00, ny = v10, nz = v20;
  if (l1 < l0) { nx = v01; ny = v11; nz = v21; }
  if (l2 < fminf(l0, l1)) { nx = v02; ny = v12; nz = v22; }
  float lo = fminf(l0, fminf(l1, l2)), hi = fmaxf(l0, fmaxf(l1, l2));
  float mid = (l0 + l1 + l2) - lo - hi;
  mid = fminf(fmaxf(mid, lo), hi);
  w[0] = lo * scale;
  w[1] = mid * scale;
  w[2] = hi * scale;
  // (w0 + w1) + w2 with one rounding per operation: left to FMA contraction, the sum would round differently in
  // each caller's inlined copy
  curv = w[0] / __fadd_rn(__fadd_rn(w[0], w[1]), w[2]);
  if (tiny) {
    w[0] *= 0x1p-64f;
    w[1] *= 0x1p-64f;
    w[2] *= 0x1p-64f;
  }
  const float rn = rsqrtf(nx * nx + ny * ny + nz * nz);
  n[0] = nx * rn;
  n[1] = ny * rn;
  n[2] = nz * rn;
}

// The smallest eigenpair alone (w and n as above).
__device__ __forceinline__ void sym3_smallest(const float (&cv)[6], float (&w)[3], float (&n)[3]) {
  float curv;
  sym3_smallest(cv, w, n, curv);
}

}  // namespace cb
