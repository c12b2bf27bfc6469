// Warp-cooperative 6x6 solve of the Gauss-Newton normal equations (product code, sm_90a): the same elimination as
// la::solve6 (solve_core.hpp: partial pivoting, one reciprocal per pivot, back substitution in the same order) with
// the augmented matrix spread over the lanes of ONE warp instead of a local-memory array of one thread. In the
// single-thread epilogue of a device-resident ICP iteration the serial version was a chain of dependent
// local-memory accesses; here every step is a handful of
// shuffles and the six divisions are the critical path.
#pragma once
#include "cb_internal.hpp"

namespace cb {

// Lane l holds column j = l % 8 (j < 7 used; column 6 = right-hand side) of rows i0 = l / 8 (register v0) and
// i0 + 4 (register v1; rows 4 and 5 only). All 32 lanes must call; every lane returns the same x[6] / flag.
__device__ __forceinline__ bool solve6_warp(const double* __restrict__ s28, int lane, double (&x)[6]) {
  const int j = lane & 7, i0 = lane >> 3;
  auto ut6 = [](int r, int c) { return r <= c ? r * 6 - (r * (r - 1)) / 2 + (c - r) : c * 6 - (c * (c - 1)) / 2 + (r - c); };
  auto entry = [&](int r, int c) -> double {
    if (r >= 6 || c >= 7) return 0.0;
    return c == 6 ? s28[22 + r] : s28[1 + ut6(r, c)];
  };
  double v0 = entry(i0, j), v1 = entry(i0 + 4, j);
  // M[r][c] as seen by every lane (r, c warp-uniform)
  auto get = [&](int r, int c) -> double {
    const double a = __shfl_sync(0xffffffffu, v0, (r & 3) * 8 + c);
    const double b = __shfl_sync(0xffffffffu, v1, (r & 3) * 8 + c);
    return (r < 4) ? a : b;
  };
  bool ok = true;
  double rp[6];
#pragma unroll
  for (int k = 0; k < 6; k++) {
    // partial pivoting: first row of maximal |M[r][k]|, r >= k
    int piv = k;
    double best = fabs(get(k, k));
#pragma unroll
    for (int r = k + 1; r < 6; r++) {
      const double c = fabs(get(r, k));
      if (c > best) {
        best = c;
        piv = r;
      }
    }
    // rows k and piv, my column
    const double rowk = get(k, j), rowp = get(piv, j);
    if (piv != k) {
      if (i0 == (k & 3)) {
        if (k < 4) v0 = rowp; else v1 = rowp;
      }
      if (i0 == (piv & 3)) {
        if (piv < 4) v0 = rowk; else v1 = rowk;
      }
    }
    const double mkj = (piv != k) ? rowp : rowk;  // M[k][j] after the swap
    const double d = __shfl_sync(0xffffffffu, mkj, (lane & ~7) + k);  // M[k][k] (any row group holds the pivot row now)
    if (d == 0.0 || !(d == d)) {
      ok = false;
      rp[k] = 0.0;
      continue;
    }
    rp[k] = 1.0 / d;
    // M[i][j] -= (M[i][k] * rp) * M[k][j] for my rows i > k, columns j >= k
    const double f0 = __shfl_sync(0xffffffffu, v0, (lane & ~7) + k) * rp[k];
    const double f1 = __shfl_sync(0xffffffffu, v1, (lane & ~7) + k) * rp[k];
    if (j >= k) {
      if (i0 > k) v0 -= f0 * mkj;
      if (i0 + 4 > k && i0 + 4 < 6) v1 -= f1 * mkj;
    }
  }
#pragma unroll
  for (int i = 5; i >= 0; i--) {
    double s = get(i, 6);
#pragma unroll
    for (int c = i + 1; c < 6; c++) s -= get(i, c) * x[c];
    x[i] = s * rp[i];
  }
  return ok;
}

}  // namespace cb
