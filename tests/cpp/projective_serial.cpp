// Serial C++ restatement of the projective correspondence search (DESIGN §4.21), compiled with -ffp-contract=off: the
// loops of CorrespondenceSearchProjective::find_correspondences_ (correspondence_search_projective.hpp:156-209) and of
// pointsToIndexMap, one point at a time. The numpy restatement (tests/projective_ref.py) is pinned against this program
// bit for bit.
//
//   projective_serial in out
//
// in:  u64 n_dst, n_src, w, h; i32 has_extrinsics; f32 max_d2; f32 K[9] (row-major), T[12], E[12] ([R | t] row-major);
//      f32 dst[3 n_dst], src[3 n_src]
// out: u64 count; then count records of (u64 first, u64 second, f32 value)
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <limits>
#include <vector>

namespace {

template <class T>
T get(FILE* f) {
  T v;
  if (std::fread(&v, sizeof(T), 1, f) != 1) throw 1;
  return v;
}

std::vector<float> arr(FILE* f, size_t n) {
  std::vector<float> v(n);
  if (n && std::fread(v.data(), sizeof(float), n, f) != n) throw 1;
  return v;
}

// Eigen's dot of two 3-vectors: (a0 b0 + a1 b1) + a2 b2
float dot(const float* a, const float* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

struct Camera {
  const float* K;
  bool extr;
  float L[9], tr[3];  // extrinsics.inverse(): linear R^T, translation -(R^T t)
  size_t w, h;

  // the pixel p lands in, or false; z = its camera-frame depth
  bool pixel(const float* p, size_t& x, size_t& y, float& z) const {
    float c[3] = {p[0], p[1], p[2]};
    if (extr)
      for (int i = 0; i < 3; i++) c[i] = dot(L + 3 * i, p) + tr[i];
    if (!(c[2] > 0.0f)) return false;
    const float inv_z = 1.0f / c[2];
    const float fx = inv_z * dot(K, c), fy = inv_z * dot(K + 3, c);
    if (!std::isfinite(fx) || !std::isfinite(fy)) return false;
    // llround only where its value is representable: anything outside (-1, w + 1) x (-1, h + 1) is off the image anyway
    if (!(fx > -1.0f && fy > -1.0f && (double)fx < (double)w + 1.0 && (double)fy < (double)h + 1.0)) return false;
    const long long xi = std::llround(fx), yi = std::llround(fy);
    if (xi < 0 || yi < 0 || (size_t)xi >= w || (size_t)yi >= h) return false;
    x = (size_t)xi;
    y = (size_t)yi;
    z = c[2];
    return true;
  }
};

}  // namespace

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 2;
  const uint64_t nd = get<uint64_t>(in), ns = get<uint64_t>(in), w = get<uint64_t>(in), h = get<uint64_t>(in);
  const int has_e = get<int32_t>(in);
  const float max_d2 = get<float>(in);
  const std::vector<float> K = arr(in, 9), T = arr(in, 12), E = arr(in, 12), dst = arr(in, 3 * nd), src = arr(in, 3 * ns);
  std::fclose(in);
  Camera cam;
  cam.K = K.data();
  cam.extr = has_e != 0;
  cam.w = w;
  cam.h = h;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) cam.L[3 * i + j] = E[4 * j + i];
  for (int i = 0; i < 3; i++) {
    const float t[3] = {E[3], E[7], E[11]};
    cam.tr[i] = -dot(cam.L + 3 * i, t);
  }
  // pointsToIndexMap: in index order, a point takes a pixel from a strictly farther one (ties keep the lower index)
  const size_t empty = std::numeric_limits<size_t>::max();
  std::vector<size_t> map(w * h, empty);
  std::vector<float> depth(w * h, 0.0f);
  for (size_t j = 0; j < nd; j++) {
    size_t x, y;
    float z;
    if (!cam.pixel(&dst[3 * j], x, y, z)) continue;
    const size_t k = y * w + x;
    if (map[k] == empty || z < depth[k]) {
      map[k] = j;
      depth[k] = z;
    }
  }
  FILE* out = std::fopen(argv[2], "wb");
  if (!out) return 2;
  std::vector<uint64_t> first, second;
  std::vector<float> value;
  for (size_t i = 0; i < ns; i++) {
    const float* s = &src[3 * i];
    float q[3];
    for (int r = 0; r < 3; r++) q[r] = (T[4 * r] * s[0] + (T[4 * r + 1] * s[1] + T[4 * r + 2] * s[2])) + T[4 * r + 3];
    size_t x, y;
    float z;
    if (!cam.pixel(q, x, y, z)) continue;
    const size_t ind = map[y * w + x];
    if (ind == empty) continue;
    const float d0 = q[0] - dst[3 * ind], d1 = q[1] - dst[3 * ind + 1], d2 = q[2] - dst[3 * ind + 2];
    const float v = (d0 * d0 + d1 * d1) + d2 * d2;
    if (!(v < max_d2)) continue;
    first.push_back(ind);
    second.push_back(i);
    value.push_back(v);
  }
  const uint64_t m = first.size();
  std::fwrite(&m, sizeof(m), 1, out);
  for (size_t k = 0; k < m; k++) {
    std::fwrite(&first[k], sizeof(uint64_t), 1, out);
    std::fwrite(&second[k], sizeof(uint64_t), 1, out);
    std::fwrite(&value[k], sizeof(float), 1, out);
  }
  std::fclose(out);
  return 0;
}
