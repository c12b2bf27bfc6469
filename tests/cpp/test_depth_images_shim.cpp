// The C++ drop-ins of core/image_point_cloud_conversions.hpp and PointCloud3f's image constructors, run on the device;
// tests/test_depth_images_shims.py compares every output with the C ABI through capi bit for bit.
//
//   test_depth_images_shim in.bin out.bin
//   in:  int64 w, h, raw_f32, truncated, n; float32 scale, max_depth, K [9] row-major, T [12] row-major [R | t];
//        raw depth [h x w] (unsigned short or float); rgb [h x w x 3] bytes; points [n x 3]; colors [n x 3]
//   out: for depthImageToPoints, depthImageToPointsNormals, RGBDImagesToPointsColors and
//        RGBDImagesToPointsNormalsColors, each without then with extrinsics, keep_invalid false then true: int64 count
//        and the float32 points, normals, colors it returns; then the same records of PointCloud3f(depth, ..., normals)
//        and PointCloud3f::fromRGBDImages(..., no normals); then pointsToDepthImage, pointsColorsToRGBDImages (depth,
//        rgb) and pointsToIndexMap<float, uint32_t> and <float, size_t>, each without then with extrinsics.
#include <cilantro/utilities/point_cloud.hpp>

#include <cstdint>
#include <cstdio>
#include <vector>

static FILE* out_file = nullptr;

template <class T>
static void put(const T* p, size_t n) {
  if (n) std::fwrite(p, sizeof(T), n, out_file);
}

static void record(const cilantro::VectorSet3f& p, const cilantro::VectorSet3f* n, const cilantro::VectorSet3f* c) {
  const int64_t m = (int64_t)p.cols();
  put(&m, 1);
  put(p.data(), 3 * p.cols());
  if (n) put(n->data(), 3 * n->cols());
  if (c) put(c->data(), 3 * c->cols());
}

template <class Raw, class Conv>
static void run(const Conv& conv, size_t w, size_t h, const cilantro::b200::Intrinsics3f& K,
                const cilantro::RigidTransform3f& T, const std::vector<Raw>& depth, const std::vector<uint8_t>& rgb,
                const cilantro::VectorSet3f& pts, const cilantro::VectorSet3f& cols) {
  using namespace cilantro;
  for (int ext = 0; ext < 2; ext++)
    for (int keep = 0; keep < 2; keep++) {
      VectorSet3f p, n, c;
      if (ext) depthImageToPoints(depth.data(), conv, w, h, K, T, p, keep);
      else depthImageToPoints(depth.data(), conv, w, h, K, p, keep);
      record(p, nullptr, nullptr);
      if (ext) depthImageToPointsNormals(depth.data(), conv, w, h, K, T, p, n, keep);
      else depthImageToPointsNormals(depth.data(), conv, w, h, K, p, n, keep);
      record(p, &n, nullptr);
      if (ext) RGBDImagesToPointsColors(rgb.data(), depth.data(), conv, w, h, K, T, p, c, keep);
      else RGBDImagesToPointsColors(rgb.data(), depth.data(), conv, w, h, K, p, c, keep);
      record(p, nullptr, &c);
      if (ext) RGBDImagesToPointsNormalsColors(rgb.data(), depth.data(), conv, w, h, K, T, p, n, c, keep);
      else RGBDImagesToPointsNormalsColors(rgb.data(), depth.data(), conv, w, h, K, p, n, c, keep);
      record(p, &n, &c);
    }
  const PointCloud3f a(depth.data(), conv, w, h, K, false, true);
  record(a.points, &a.normals, nullptr);
  PointCloud3f b;
  b.fromRGBDImages(rgb.data(), depth.data(), conv, w, h, K);
  record(b.points, nullptr, &b.colors);
  std::vector<Raw> d(w * h);
  std::vector<uint8_t> im(3 * w * h);
  std::vector<uint32_t> i32(w * h);
  std::vector<size_t> i64(w * h);
  for (int ext = 0; ext < 2; ext++) {
    if (ext) pointsToDepthImage(pts, T, K, conv, d.data(), w, h);
    else pointsToDepthImage(pts, K, conv, d.data(), w, h);
    put(d.data(), d.size());
    if (ext) pointsColorsToRGBDImages(pts, cols, T, K, conv, im.data(), d.data(), w, h);
    else pointsColorsToRGBDImages(pts, cols, K, conv, im.data(), d.data(), w, h);
    put(d.data(), d.size());
    put(im.data(), im.size());
    if (ext) pointsToIndexMap(pts, T, K, i32.data(), w, h);
    else pointsToIndexMap(pts, K, i32.data(), w, h);
    put(i32.data(), i32.size());
    if (ext) pointsToIndexMap<float>(pts, T, K, i64.data(), w, h);
    else pointsToIndexMap<float>(pts, K, i64.data(), w, h);
    put(i64.data(), i64.size());
  }
}

template <class T>
static bool get(FILE* f, T* p, size_t n) {
  return std::fread(p, sizeof(T), n, f) == n;
}

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  int64_t hdr[5];
  float sc[2], Km[9], Tm[12];
  if (!get(f, hdr, 5) || !get(f, sc, 2) || !get(f, Km, 9) || !get(f, Tm, 12)) return 2;
  const size_t w = (size_t)hdr[0], h = (size_t)hdr[1], n = (size_t)hdr[4];
  const bool f32 = hdr[2] != 0, truncated = hdr[3] != 0;
  std::vector<uint16_t> d16(f32 ? 0 : w * h);
  std::vector<float> d32(f32 ? w * h : 0);
  if (f32 ? !get(f, d32.data(), w * h) : !get(f, d16.data(), w * h)) return 2;
  std::vector<uint8_t> rgb(3 * w * h);
  cilantro::VectorSet3f pts(3, n), cols(3, n);
  if (!get(f, rgb.data(), rgb.size()) || !get(f, pts.data(), 3 * n) || !get(f, cols.data(), 3 * n)) return 2;
  std::fclose(f);
  out_file = std::fopen(argv[2], "wb");
  if (!out_file) return 2;
  const cilantro::b200::Intrinsics3f K(Km);
  const cilantro::RigidTransform3f T(Tm);
  if (f32 && truncated)
    run(cilantro::TruncatedDepthValueConverter<float, float>(sc[0], sc[1]), w, h, K, T, d32, rgb, pts, cols);
  else if (f32)
    run(cilantro::DepthValueConverter<float, float>(sc[0]), w, h, K, T, d32, rgb, pts, cols);
  else if (truncated)
    run(cilantro::TruncatedDepthValueConverter<unsigned short, float>(sc[0], sc[1]), w, h, K, T, d16, rgb, pts, cols);
  else
    run(cilantro::DepthValueConverter<unsigned short, float>(sc[0]), w, h, K, T, d16, rgb, pts, cols);
  std::fclose(out_file);
  return 0;
}
