// Test harness for the hypothesis-plane fit (cilantro_b200/csrc/plane_fit.hpp); tests/test_gpu_ransac_plane.py builds
// it with nvcc and the library's flags (the fit runs inside a kernel, as in plane_fit_kernel) and with g++ -x c++ (the
// host build), and checks that both give the same bits.
//
//   plane_fit_harness <in.bin> <out.bin>
// Records are packed float32: in 10 = 9 coordinates (3 points) + the point count; out 4 = (n0, n1, n2, d).
#include <cstdio>
#include <vector>

#include "plane_fit.hpp"

#if defined(__CUDACC__)
__global__ void fit_kernel(const float* in, float* out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) cb::plane::fit(in + 10 * (size_t)i, (int)in[10 * (size_t)i + 9], out + 4 * (size_t)i);
}
#endif

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 3;
  std::vector<float> in;
  float buf[10];
  while (std::fread(buf, sizeof(float), 10, f) == 10) in.insert(in.end(), buf, buf + 10);
  std::fclose(f);
  const int n = (int)(in.size() / 10);
  std::vector<float> out(4 * (size_t)n);
#if defined(__CUDACC__)
  float *d_in = nullptr, *d_out = nullptr;
  if (cudaMalloc(&d_in, in.size() * sizeof(float) + 4) != cudaSuccess) return 4;
  if (cudaMalloc(&d_out, out.size() * sizeof(float) + 4) != cudaSuccess) return 4;
  cudaMemcpy(d_in, in.data(), in.size() * sizeof(float), cudaMemcpyHostToDevice);
  fit_kernel<<<(n + 127) / 128, 128>>>(d_in, d_out, n);
  if (cudaMemcpy(out.data(), d_out, out.size() * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess) return 5;
  cudaFree(d_in);
  cudaFree(d_out);
#else
  for (int i = 0; i < n; i++) cb::plane::fit(&in[10 * (size_t)i], (int)in[10 * (size_t)i + 9], &out[4 * (size_t)i]);
#endif
  f = std::fopen(argv[2], "wb");
  if (!f) return 3;
  std::fwrite(out.data(), sizeof(float), out.size(), f);
  std::fclose(f);
  return 0;
}
