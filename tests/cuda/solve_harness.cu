// Test harness for the O(1) solves of the product (tests/test_solve_device.py builds and drives it).
//
// Built with nvcc and the library's flags, it runs the shipped headers inside kernels: la::nearest_rotation,
// sc::kabsch_from_moments, la::solve6 and solve6_warp (solve_core.hpp, solve_warp.cuh) and sym3_smallest
// (sym3_eigen.cuh). Built with g++ (-x c++), it runs the host-capable part (solve_core.hpp) on the CPU.
//
//   solve_harness <mode> <in.bin> <out.bin>
// Records are packed float64 (sym3: float32), one per case:
//   rotation  in  9  sigma (row-major)          out 20  R (flip col 2), R (flip col 0), polar taken, 0
//   kabsch    in 16  moments about zero pivots   out 13  T (3x4), ok
//   solve6    in 28  {n, upper AtA (21), Atb}    out 14  x, ok (la::solve6) | device: x, ok (solve6_warp)
//                                                        | host: the first half again
//   sym3      in  6  xx xy xz yy yz zz (fp32)    out  7  w (ascending), n, curvature (fp32)   [device only]
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "solve_core.hpp"
#if defined(__CUDACC__)
#include "solve_warp.cuh"
#include "sym3_eigen.cuh"
#endif

namespace {

CB_HD void run_rotation(const double* in, double* out) {
  cb::la::Mat3 A;
  for (int i = 0; i < 9; i++) A.m[i / 3][i % 3] = in[i];
  const cb::la::Mat3 R2 = cb::la::nearest_rotation(A, 2), R0 = cb::la::nearest_rotation(A, 0);
  cb::la::Mat3 Q;
  const bool polar = cb::la::polar_rotation(A, Q);
  for (int i = 0; i < 9; i++) {
    out[i] = R2.m[i / 3][i % 3];
    out[9 + i] = R0.m[i / 3][i % 3];
  }
  out[18] = polar ? 1.0 : 0.0;
  out[19] = 0.0;
}

CB_HD void run_kabsch(const double* in, double* out) {
  float T[12];
  const bool ok = cb::sc::kabsch_from_moments(in, nullptr, nullptr, T);
  for (int i = 0; i < 12; i++) out[i] = T[i];
  out[12] = ok ? 1.0 : 0.0;
}

CB_HD void run_solve6(const double* in, double* out) {
  double x[6];
  const bool ok = cb::sc::gauss_newton_solve(in, x);
  for (int i = 0; i < 6; i++) out[i] = x[i];
  out[6] = ok ? 1.0 : 0.0;
}

#if defined(__CUDACC__)
__global__ void rotation_kernel(const double* in, double* out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) run_rotation(in + 9 * (size_t)i, out + 20 * (size_t)i);
}

__global__ void kabsch_kernel(const double* in, double* out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) run_kabsch(in + 16 * (size_t)i, out + 13 * (size_t)i);
}

// one warp per case: lane 0 runs the serial la::solve6, the whole warp solve6_warp
__global__ void solve6_kernel(const double* in, double* out, int n) {
  const int c = blockIdx.x;
  if (c >= n) return;
  const double* s = in + 28 * (size_t)c;
  double* o = out + 14 * (size_t)c;
  if (threadIdx.x == 0) run_solve6(s, o);
  double x[6];
  const bool ok = cb::solve6_warp(s, (int)threadIdx.x, x);
  if (threadIdx.x == 0) {
    for (int i = 0; i < 6; i++) o[7 + i] = x[i];
    o[13] = ok ? 1.0 : 0.0;
  }
}

__global__ void sym3_kernel(const float* in, float* out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float cv[6], w[3], nv[3], curv;
  for (int k = 0; k < 6; k++) cv[k] = in[6 * (size_t)i + k];
  cb::sym3_smallest(cv, w, nv, curv);
  float* o = out + 7 * (size_t)i;
  for (int k = 0; k < 3; k++) {
    o[k] = w[k];
    o[3 + k] = nv[k];
  }
  o[6] = curv;
}

#define CHECK(call)                                                                 \
  do {                                                                              \
    cudaError_t e__ = (call);                                                       \
    if (e__ != cudaSuccess) {                                                       \
      fprintf(stderr, "%s:%d: %s\n", __FILE__, __LINE__, cudaGetErrorString(e__)); \
      exit(2);                                                                      \
    }                                                                               \
  } while (0)

template <class T, class Launch>
void run_device(const std::vector<char>& in, size_t in_rec, size_t out_rec, size_t n, std::vector<char>& out,
                Launch launch) {
  T *d_in = nullptr, *d_out = nullptr;
  CHECK(cudaMalloc(&d_in, in.size() + 1));
  CHECK(cudaMalloc(&d_out, n * out_rec * sizeof(T) + 1));
  CHECK(cudaMemcpy(d_in, in.data(), in.size(), cudaMemcpyHostToDevice));
  launch(d_in, d_out, (int)n);
  CHECK(cudaGetLastError());
  CHECK(cudaDeviceSynchronize());
  out.resize(n * out_rec * sizeof(T));
  CHECK(cudaMemcpy(out.data(), d_out, out.size(), cudaMemcpyDeviceToHost));
  CHECK(cudaFree(d_in));
  CHECK(cudaFree(d_out));
  (void)in_rec;
}
#endif

}  // namespace

int main(int argc, char** argv) {
  if (argc != 4) {
    fprintf(stderr, "usage: %s rotation|kabsch|solve6|sym3 in.bin out.bin\n", argv[0]);
    return 1;
  }
  const char* mode = argv[1];
  FILE* f = fopen(argv[2], "rb");
  if (!f) return 1;
  std::vector<char> in;
  char buf[1 << 16];
  size_t got;
  while ((got = fread(buf, 1, sizeof(buf), f)) > 0) in.insert(in.end(), buf, buf + got);
  fclose(f);
  std::vector<char> out;
  const bool sym3 = !strcmp(mode, "sym3");
  const size_t in_rec = !strcmp(mode, "rotation") ? 9 : !strcmp(mode, "kabsch") ? 16 : !strcmp(mode, "solve6") ? 28 : 6;
  const size_t out_rec = !strcmp(mode, "rotation") ? 20 : !strcmp(mode, "kabsch") ? 13 : !strcmp(mode, "solve6") ? 14 : 7;
  const size_t n = in.size() / (in_rec * (sym3 ? sizeof(float) : sizeof(double)));
#if defined(__CUDACC__)
  if (!strcmp(mode, "rotation")) {
    run_device<double>(in, in_rec, out_rec, n, out, [](const double* a, double* b, int m) {
      rotation_kernel<<<(m + 63) / 64, 64>>>(a, b, m);
    });
  } else if (!strcmp(mode, "kabsch")) {
    run_device<double>(in, in_rec, out_rec, n, out, [](const double* a, double* b, int m) {
      kabsch_kernel<<<(m + 63) / 64, 64>>>(a, b, m);
    });
  } else if (!strcmp(mode, "solve6")) {
    run_device<double>(in, in_rec, out_rec, n, out, [](const double* a, double* b, int m) {
      if (m) solve6_kernel<<<m, 32>>>(a, b, m);
    });
  } else if (sym3) {
    run_device<float>(in, in_rec, out_rec, n, out, [](const float* a, float* b, int m) {
      sym3_kernel<<<(m + 63) / 64, 64>>>(a, b, m);
    });
  } else {
    return 1;
  }
#else
  if (sym3) {
    fprintf(stderr, "sym3 runs on the device only\n");
    return 1;
  }
  const double* src = reinterpret_cast<const double*>(in.data());
  out.assign(n * out_rec * sizeof(double), 0);
  double* dst = reinterpret_cast<double*>(out.data());
  for (size_t i = 0; i < n; i++) {
    if (!strcmp(mode, "rotation")) {
      run_rotation(src + in_rec * i, dst + out_rec * i);
    } else if (!strcmp(mode, "kabsch")) {
      run_kabsch(src + in_rec * i, dst + out_rec * i);
    } else if (!strcmp(mode, "solve6")) {
      run_solve6(src + in_rec * i, dst + out_rec * i);
      memcpy(dst + out_rec * i + 7, dst + out_rec * i, 7 * sizeof(double));
    } else {
      return 1;
    }
  }
#endif
  FILE* g = fopen(argv[3], "wb");
  if (!g) return 1;
  fwrite(out.data(), 1, out.size(), g);
  fclose(g);
  return 0;
}
