// Serial C++ restatement of the depth-image <-> cloud contract (DESIGN §4.20), compiled with -ffp-contract=off: the
// reference's loops run one pixel / one point at a time, which is the result the device must reproduce. The numpy
// restatement (tests/depth_images_ref.py) is pinned against this program bit for bit.
//
//   depth_images_serial back   in out   (image -> points)
//   depth_images_serial render in out   (points -> depth / RGB-D image / index map)
//
// Input files are little-endian records as written by tests/test_depth_images_ref.py.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <limits>
#include <string>
#include <vector>

namespace {

struct Reader {
  FILE* f;
  template <class T>
  T get() {
    T v;
    if (std::fread(&v, sizeof(T), 1, f) != 1) throw 1;
    return v;
  }
  template <class T>
  std::vector<T> arr(size_t n) {
    std::vector<T> v(n);
    if (n && std::fread(v.data(), sizeof(T), n, f) != n) throw 1;
    return v;
  }
};

template <class T>
void put(FILE* f, const std::vector<T>& v) {
  if (!v.empty()) std::fwrite(v.data(), sizeof(T), v.size(), f);
}

float dot(const float* a, float b0, float b1, float b2) { return (a[0] * b0 + a[1] * b1) + a[2] * b2; }

// Eigen 3.4's inverse of a fixed 3 x 3 (row-major here)
void inverse3(const float* m, float* inv) {
  auto at = [&](int r, int c) { return m[3 * r + c]; };
  auto cof = [&](int i, int j) {
    const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
    return at(i1, j1) * at(i2, j2) - at(i1, j2) * at(i2, j1);
  };
  const float c0 = cof(0, 0), c1 = cof(1, 0), c2 = cof(2, 0);
  const float det = (c0 * at(0, 0) + c1 * at(1, 0)) + c2 * at(2, 0);
  const float invdet = 1.0f / det;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) inv[3 * i + j] = cof(j, i) * invdet;
}

int back(Reader& in, FILE* out) {
  const uint64_t w = in.get<uint64_t>(), h = in.get<uint64_t>();
  const int32_t f32 = in.get<int32_t>(), truncated = in.get<int32_t>();
  const float scale = in.get<float>(), max_depth = in.get<float>();
  const std::vector<float> K = in.arr<float>(9);
  const int32_t has_extr = in.get<int32_t>();
  const std::vector<float> T = in.arr<float>(12);
  const int32_t normals = in.get<int32_t>(), keep_invalid = in.get<int32_t>(), has_rgb = in.get<int32_t>();
  const size_t npix = w * h;
  std::vector<float> zs(npix);
  if (f32) {
    const std::vector<float> raw = in.arr<float>(npix);
    for (size_t k = 0; k < npix; k++) zs[k] = (1.0f / scale) * raw[k];
  } else {
    const std::vector<uint16_t> raw = in.arr<uint16_t>(npix);
    for (size_t k = 0; k < npix; k++) zs[k] = (1.0f / scale) * static_cast<float>(raw[k]);
  }
  if (truncated)
    for (float& z : zs) z = z < max_depth ? z : 0.0f;
  const std::vector<uint8_t> rgb = has_rgb ? in.arr<uint8_t>(3 * npix) : std::vector<uint8_t>();
  float Ki[9], A[9];
  inverse3(K.data(), Ki);
  std::memcpy(A, Ki, sizeof(A));
  bool post = has_extr != 0;
  float R[9], t[3];
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) R[3 * i + j] = T[4 * i + j];
    t[i] = T[4 * i + 3];
  }
  if (post && keep_invalid && !normals) {
    // (extrinsics * intrinsics_inv) * v; the isometry maps the columns of intrinsics_inv as points
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) A[3 * i + j] = t[i] + dot(R + 3 * i, Ki[j], Ki[3 + j], Ki[6 + j]);
    post = false;
  }
  std::vector<float> p(3 * npix), n(3 * npix, std::numeric_limits<float>::quiet_NaN()), c(3 * npix);
  for (size_t y = 0; y < h; y++)
    for (size_t x = 0; x < w; x++) {
      const size_t k = y * w + x;
      const float z = zs[k], v0 = z * x, v1 = z * y;
      for (int i = 0; i < 3; i++) p[3 * k + i] = dot(A + 3 * i, v0, v1, z);
      if (has_rgb)
        for (int i = 0; i < 3; i++) c[3 * k + i] = (1.0f / 255.0f) * static_cast<float>(rgb[3 * k + i]);
    }
  if (normals && w >= 3 && h >= 3)
    for (size_t y = 1; y < h - 1; y++)
      for (size_t x = 1; x < w - 1; x++) {
        const size_t k = y * w + x;
        auto z = [&](size_t q) { return p[3 * q + 2]; };
        if (!(z(k) > 0 && z(k + 1) > 0 && z(k - 1) > 0 && z(k + w) > 0 && z(k - w) > 0)) continue;
        float a[3], b[3];
        for (int i = 0; i < 3; i++) {
          a[i] = p[3 * (k + w) + i] - p[3 * (k - w) + i];
          b[i] = p[3 * (k + 1) + i] - p[3 * (k - 1) + i];
        }
        float cr[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
        const float s = (cr[0] * cr[0] + cr[1] * cr[1]) + cr[2] * cr[2];
        if (s > 0) {
          const float r = std::sqrt(s);
          for (float& e : cr) e = e / r;
        }
        for (int i = 0; i < 3; i++) n[3 * k + i] = cr[i];
      }
  std::vector<float> op, on, oc;
  for (size_t k = 0; k < npix; k++) {
    const bool keep = normals ? !std::isnan(n[3 * k]) : p[3 * k + 2] > 0;
    if (!keep_invalid && !keep) continue;
    float q[3] = {p[3 * k], p[3 * k + 1], p[3 * k + 2]}, m[3] = {n[3 * k], n[3 * k + 1], n[3 * k + 2]};
    if (post) {
      const float q2[3] = {dot(R, q[0], q[1], q[2]) + t[0], dot(R + 3, q[0], q[1], q[2]) + t[1],
                           dot(R + 6, q[0], q[1], q[2]) + t[2]};
      const float m2[3] = {dot(R, m[0], m[1], m[2]), dot(R + 3, m[0], m[1], m[2]), dot(R + 6, m[0], m[1], m[2])};
      std::memcpy(q, q2, sizeof(q));
      std::memcpy(m, m2, sizeof(m));
    }
    op.insert(op.end(), q, q + 3);
    if (normals) on.insert(on.end(), m, m + 3);
    if (has_rgb) oc.insert(oc.end(), c.begin() + 3 * k, c.begin() + 3 * k + 3);
  }
  const uint64_t m = op.size() / 3;
  std::fwrite(&m, sizeof(m), 1, out);
  put(out, op);
  put(out, on);
  put(out, oc);
  return 0;
}

int render(Reader& in, FILE* out) {
  const uint64_t n = in.get<uint64_t>(), w = in.get<uint64_t>(), h = in.get<uint64_t>();
  const int32_t mode = in.get<int32_t>(), truncated = in.get<int32_t>();  // mode: 0 u16, 1 f32, 2 index map
  const float scale = in.get<float>(), max_depth = in.get<float>();
  const std::vector<float> K = in.arr<float>(9);
  const int32_t has_extr = in.get<int32_t>();
  const std::vector<float> T = in.arr<float>(12);
  const int32_t has_col = in.get<int32_t>();
  const std::vector<float> pts = in.arr<float>(3 * n);
  const std::vector<float> col = has_col ? in.arr<float>(3 * n) : std::vector<float>();
  float L[9], tr[3];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) L[3 * i + j] = T[4 * j + i];
  for (int i = 0; i < 3; i++) tr[i] = -dot(L + 3 * i, T[3], T[7], T[11]);
  const size_t npix = w * h;
  std::vector<uint16_t> d16(npix, 0);
  std::vector<float> d32(npix, 0.0f), zbuf(npix, 0.0f);
  std::vector<uint8_t> rgb(3 * npix, 0);
  std::vector<uint64_t> idx(npix, std::numeric_limits<uint64_t>::max());
  for (size_t i = 0; i < n; i++) {
    float q[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
    if (has_extr) {
      const float c[3] = {dot(L, q[0], q[1], q[2]) + tr[0], dot(L + 3, q[0], q[1], q[2]) + tr[1],
                          dot(L + 6, q[0], q[1], q[2]) + tr[2]};
      std::memcpy(q, c, sizeof(q));
    }
    if (q[2] <= 0.0f) continue;
    const float inv_z = 1.0f / q[2];
    const float fx = inv_z * dot(K.data(), q[0], q[1], q[2]), fy = inv_z * dot(K.data() + 3, q[0], q[1], q[2]);
    if (!std::isfinite(fx) || !std::isfinite(fy)) continue;
    const double rx = std::round((double)fx), ry = std::round((double)fy);
    if (rx < 0 || ry < 0 || rx >= (double)w || ry >= (double)h) continue;
    const size_t k = (size_t)ry * w + (size_t)rx;
    if (mode == 2) {
      if (idx[k] == std::numeric_limits<uint64_t>::max() || q[2] < zbuf[k]) {
        idx[k] = i;
        zbuf[k] = q[2];
      }
      continue;
    }
    if (truncated && !(q[2] < max_depth)) continue;
    const float v = scale * q[2];
    bool write;
    if (mode == 0) {
      if (!(v >= 0.0f && v < 65536.0f)) continue;
      const uint16_t raw = static_cast<uint16_t>(v);
      write = raw > 0 && (d16[k] == 0 || raw < d16[k]);
      if (write) d16[k] = raw;
    } else {
      write = v > 0.0f && (d32[k] == 0.0f || v < d32[k]);
      if (write) d32[k] = v;
    }
    if (write && has_col)
      for (int c = 0; c < 3; c++) {
        const float b = 255.0f * col[3 * i + c];
        rgb[3 * k + c] = !(b > 0.0f) ? 0 : b >= 255.0f ? 255 : static_cast<uint8_t>(b);
      }
  }
  if (mode == 2) {
    put(out, idx);
    return 0;
  }
  if (mode == 0)
    put(out, d16);
  else
    put(out, d32);
  if (has_col) put(out, rgb);
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  if (argc != 4) {
    std::fprintf(stderr, "usage: %s back|render in out\n", argv[0]);
    return 2;
  }
  FILE* fi = std::fopen(argv[2], "rb");
  FILE* fo = std::fopen(argv[3], "wb");
  if (!fi || !fo) return 2;
  Reader in{fi};
  int rc = 2;
  try {
    rc = std::string(argv[1]) == "back" ? back(in, fo) : render(in, fo);
  } catch (int) {
    std::fprintf(stderr, "short input\n");
  }
  std::fclose(fi);
  std::fclose(fo);
  return rc;
}
