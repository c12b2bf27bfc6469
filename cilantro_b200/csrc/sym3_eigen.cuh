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

__device__ __forceinline__ void sym3_smallest(const float (&cv)[6], float (&w)[3], float (&n)[3]) {
  float scale = fmaxf(fmaxf(fabsf(cv[0]), fabsf(cv[1])), fmaxf(fabsf(cv[2]), fabsf(cv[3])));
  scale = fmaxf(scale, fmaxf(fabsf(cv[4]), fabsf(cv[5])));
  if (!(scale > 0.f)) {  // zero matrix: eigenvectors = identity (and NaN input falls through as NaN below)
    w[0] = w[1] = w[2] = scale;
    n[0] = 1.f;
    n[1] = 0.f;
    n[2] = 0.f;
    return;
  }
  const float inv = 1.f / scale;
  float a00 = cv[0] * inv, a01 = cv[1] * inv, a02 = cv[2] * inv, a11 = cv[3] * inv, a12 = cv[4] * inv,
        a22 = cv[5] * inv;
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
  const float rn = rsqrtf(nx * nx + ny * ny + nz * nz);
  n[0] = nx * rn;
  n[1] = ny * rn;
  n[2] = nz * rn;
}

}  // namespace cb
