// Same include path as cilantro's core/image_point_cloud_conversions.hpp. Depth-image and RGB-D <-> cloud conversions
// on the device (cb_depth_image_to_points, cb_points_to_depth_image, cb_points_to_index_map; DESIGN §4.20):
// DepthValueConverter / TruncatedDepthValueConverter (:7-51), depthImageToPoints, depthImageToPointsNormals,
// RGBDImagesToPointsColors, RGBDImagesToPointsNormalsColors (:53-695), pointsToDepthImage, pointsColorsToRGBDImages
// and pointsToIndexMap (:697-934), each with and without extrinsics. MetricDepth is float; RawDepth is unsigned short
// or float. Intrinsics are a b200::Intrinsics3f (row-major 3 x 3), converted implicitly from an
// Eigen::Matrix<float, 3, 3> where Eigen is available. The depth and rgb buffers may be host or device memory.
#pragma once
#include <cstdint>
#include <cstring>
#include <limits>
#include <type_traits>
#include <vector>

#include "../b200_shims.hpp"

namespace cilantro {

namespace b200 {

// Row-major 3 x 3 intrinsics (the stand-in for Eigen::Ref<const Eigen::Matrix<float, 3, 3>>).
struct Intrinsics3f {
  float m[9] = {1.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 1.f};
  Intrinsics3f() = default;
  explicit Intrinsics3f(const float* row_major) { std::memcpy(m, row_major, sizeof(m)); }
  Intrinsics3f(float fx, float fy, float cx, float cy) : m{fx, 0.f, cx, 0.f, fy, cy, 0.f, 0.f, 1.f} {}
  float operator()(size_t r, size_t c) const { return m[3 * r + c]; }
  float& operator()(size_t r, size_t c) { return m[3 * r + c]; }
#ifdef CILANTRO_B200_HAS_EIGEN
  Intrinsics3f(const Eigen::Matrix<float, 3, 3>& K) {
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) m[3 * r + c] = K(r, c);
  }
#endif
};

template <typename RawDepthT, typename MetricDepthT>
struct DepthTypes {
  static_assert(std::is_same<MetricDepthT, float>::value, "cilantro_b200: float MetricDepth only");
  static_assert(std::is_same<RawDepthT, unsigned short>::value || std::is_same<RawDepthT, float>::value,
                "cilantro_b200: RawDepth must be unsigned short or float");
  static constexpr int32_t raw_type = std::is_same<RawDepthT, float>::value ? CB_DEPTH_F32 : CB_DEPTH_U16;
};

template <class DepthConverterT>
cb_depth_converter converter_of(const DepthConverterT& c) {
  cb_depth_converter r;
  r.raw_type = DepthTypes<typename DepthConverterT::RawDepth, typename DepthConverterT::MetricDepth>::raw_type;
  r.truncated = DepthConverterT::kTruncated ? 1 : 0;
  r.scale = c.scale;
  r.max_depth = c.truncation();
  return r;
}

template <class DepthConverterT>
void image_to_points(const typename DepthConverterT::RawDepth* depth_data, const unsigned char* rgb_data,
                     const DepthConverterT& conv, size_t image_w, size_t image_h, const Intrinsics3f& intrinsics,
                     const RigidTransform3f* extrinsics, VectorSet3f& points, VectorSet3f* normals,
                     VectorSet3f* colors, bool keep_invalid) {
  const cb_depth_converter c = converter_of(conv);
  const size_t npix = image_w * image_h;
  points.resize(3, npix);
  if (normals) normals->resize(3, npix);
  if (colors) colors->resize(3, npix);
  size_t count = 0;
  check(cb_depth_image_to_points(Context::get(), depth_data, rgb_data, image_w, image_h, &c, intrinsics.m,
                                 extrinsics ? extrinsics->data() : nullptr, normals ? 1 : 0, keep_invalid ? 1 : 0,
                                 points.data(), normals ? normals->data() : nullptr,
                                 colors ? colors->data() : nullptr, &count, nullptr),
        "cb_depth_image_to_points");
  points.resize(3, count);
  if (normals) normals->resize(3, count);
  if (colors) colors->resize(3, count);
}

template <class DepthConverterT>
void cloud_to_depth(const ConstVectorSetMatrixMap3f& points, const ConstVectorSetMatrixMap3f* colors,
                    const RigidTransform3f* extrinsics, const Intrinsics3f& intrinsics, const DepthConverterT& conv,
                    unsigned char* rgb_data, typename DepthConverterT::RawDepth* depth_data, size_t image_w,
                    size_t image_h) {
  const cb_depth_converter c = converter_of(conv);
  check(cb_points_to_depth_image(Context::get(), points.data(), nullptr, points.cols(),
                                 colors ? colors->data() : nullptr, intrinsics.m,
                                 extrinsics ? extrinsics->data() : nullptr, &c, image_w, image_h, depth_data,
                                 colors ? rgb_data : nullptr),
        "cb_points_to_depth_image");
}

template <typename PointT, typename IndexT>
void cloud_to_index_map(const ConstVectorSetMatrixMap3f& points, const RigidTransform3f* extrinsics,
                        const Intrinsics3f& intrinsics, IndexT* index_map_data, size_t image_w, size_t image_h) {
  static_assert(std::is_same<PointT, float>::value, "cilantro_b200: float pointsToIndexMap only");
  std::vector<uint64_t> idx(image_w * image_h);
  check(cb_points_to_index_map(Context::get(), points.data(), nullptr, points.cols(), intrinsics.m,
                               extrinsics ? extrinsics->data() : nullptr, image_w, image_h, idx.data()),
        "cb_points_to_index_map");
  for (size_t i = 0; i < idx.size(); i++)
    index_map_data[i] = idx[i] == std::numeric_limits<uint64_t>::max() ? std::numeric_limits<IndexT>::max()
                                                                        : static_cast<IndexT>(idx[i]);
}

}  // namespace b200

template <typename RawDepthT, typename MetricDepthT>
struct DepthValueConverter {
  using RawDepth = RawDepthT;
  using MetricDepth = MetricDepthT;
  static constexpr bool kTruncated = false;
  static_assert(sizeof(b200::DepthTypes<RawDepthT, MetricDepthT>) > 0, "");

  DepthValueConverter() : scale((MetricDepthT)1.0), inverseScale((MetricDepthT)1.0) {}
  DepthValueConverter(MetricDepthT mult) : scale(mult), inverseScale((MetricDepthT)1.0 / mult) {}

  inline MetricDepthT getMetricValue(RawDepthT val) const { return inverseScale * static_cast<MetricDepthT>(val); }
  inline RawDepthT getRawValue(MetricDepthT val) const { return static_cast<RawDepthT>(scale * val); }
  MetricDepthT truncation() const { return (MetricDepthT)0; }

  const MetricDepthT scale;
  const MetricDepthT inverseScale;
};

template <typename RawDepthT, typename MetricDepthT>
struct TruncatedDepthValueConverter {
  using RawDepth = RawDepthT;
  using MetricDepth = MetricDepthT;
  static constexpr bool kTruncated = true;
  static_assert(sizeof(b200::DepthTypes<RawDepthT, MetricDepthT>) > 0, "");

  TruncatedDepthValueConverter()
      : scale((MetricDepthT)1.0), inverseScale((MetricDepthT)1.0), maxDepth(std::numeric_limits<MetricDepthT>::max()) {}
  TruncatedDepthValueConverter(MetricDepthT mult, MetricDepthT thresh)
      : scale(mult), inverseScale((MetricDepthT)1.0 / mult), maxDepth(thresh) {}

  inline MetricDepthT getMetricValue(RawDepthT val) const {
    const MetricDepthT res = inverseScale * static_cast<MetricDepthT>(val);
    return (res < maxDepth) ? res : (MetricDepthT)0.0;
  }
  inline RawDepthT getRawValue(MetricDepthT val) const {
    return (val < maxDepth) ? static_cast<RawDepthT>(scale * val) : (RawDepthT)0;
  }
  MetricDepthT truncation() const { return maxDepth; }

  const MetricDepthT scale;
  const MetricDepthT inverseScale;
  const MetricDepthT maxDepth;
};

// ---- image -> cloud (:53-695) ------------------------------------------------------------------------------------
template <class DepthConverterT>
void depthImageToPoints(const typename DepthConverterT::RawDepth* depth_data, const DepthConverterT& depth_converter,
                        size_t image_w, size_t image_h, const b200::Intrinsics3f& intrinsics, VectorSet3f& points,
                        bool keep_invalid = false) {
  b200::image_to_points(depth_data, nullptr, depth_converter, image_w, image_h, intrinsics, nullptr, points, nullptr,
                        nullptr, keep_invalid);
}

template <class DepthConverterT>
void depthImageToPoints(const typename DepthConverterT::RawDepth* depth_data, const DepthConverterT& depth_converter,
                        size_t image_w, size_t image_h, const b200::Intrinsics3f& intrinsics,
                        const RigidTransform3f& extrinsics, VectorSet3f& points, bool keep_invalid = false) {
  b200::image_to_points(depth_data, nullptr, depth_converter, image_w, image_h, intrinsics, &extrinsics, points,
                        nullptr, nullptr, keep_invalid);
}

template <class DepthConverterT>
void depthImageToPointsNormals(const typename DepthConverterT::RawDepth* depth_data,
                               const DepthConverterT& depth_converter, size_t image_w, size_t image_h,
                               const b200::Intrinsics3f& intrinsics, VectorSet3f& points, VectorSet3f& normals,
                               bool keep_invalid = false) {
  b200::image_to_points(depth_data, nullptr, depth_converter, image_w, image_h, intrinsics, nullptr, points, &normals,
                        nullptr, keep_invalid);
}

template <class DepthConverterT>
void depthImageToPointsNormals(const typename DepthConverterT::RawDepth* depth_data,
                               const DepthConverterT& depth_converter, size_t image_w, size_t image_h,
                               const b200::Intrinsics3f& intrinsics, const RigidTransform3f& extrinsics,
                               VectorSet3f& points, VectorSet3f& normals, bool keep_invalid = false) {
  b200::image_to_points(depth_data, nullptr, depth_converter, image_w, image_h, intrinsics, &extrinsics, points,
                        &normals, nullptr, keep_invalid);
}

template <class DepthConverterT>
void RGBDImagesToPointsColors(const unsigned char* rgb_data, const typename DepthConverterT::RawDepth* depth_data,
                              const DepthConverterT& depth_converter, size_t image_w, size_t image_h,
                              const b200::Intrinsics3f& intrinsics, VectorSet3f& points, VectorSet3f& colors,
                              bool keep_invalid = false) {
  b200::image_to_points(depth_data, rgb_data, depth_converter, image_w, image_h, intrinsics, nullptr, points, nullptr,
                        &colors, keep_invalid);
}

template <class DepthConverterT>
void RGBDImagesToPointsColors(const unsigned char* rgb_data, const typename DepthConverterT::RawDepth* depth_data,
                              const DepthConverterT& depth_converter, size_t image_w, size_t image_h,
                              const b200::Intrinsics3f& intrinsics, const RigidTransform3f& extrinsics,
                              VectorSet3f& points, VectorSet3f& colors, bool keep_invalid = false) {
  b200::image_to_points(depth_data, rgb_data, depth_converter, image_w, image_h, intrinsics, &extrinsics, points,
                        nullptr, &colors, keep_invalid);
}

template <class DepthConverterT>
void RGBDImagesToPointsNormalsColors(const unsigned char* rgb_data,
                                     const typename DepthConverterT::RawDepth* depth_data,
                                     const DepthConverterT& depth_converter, size_t image_w, size_t image_h,
                                     const b200::Intrinsics3f& intrinsics, VectorSet3f& points, VectorSet3f& normals,
                                     VectorSet3f& colors, bool keep_invalid = false) {
  b200::image_to_points(depth_data, rgb_data, depth_converter, image_w, image_h, intrinsics, nullptr, points, &normals,
                        &colors, keep_invalid);
}

template <class DepthConverterT>
void RGBDImagesToPointsNormalsColors(const unsigned char* rgb_data,
                                     const typename DepthConverterT::RawDepth* depth_data,
                                     const DepthConverterT& depth_converter, size_t image_w, size_t image_h,
                                     const b200::Intrinsics3f& intrinsics, const RigidTransform3f& extrinsics,
                                     VectorSet3f& points, VectorSet3f& normals, VectorSet3f& colors,
                                     bool keep_invalid = false) {
  b200::image_to_points(depth_data, rgb_data, depth_converter, image_w, image_h, intrinsics, &extrinsics, points,
                        &normals, &colors, keep_invalid);
}

// ---- cloud -> image (:697-934) -----------------------------------------------------------------------------------
template <class DepthConverterT>
void pointsToDepthImage(const ConstVectorSetMatrixMap3f& points, const b200::Intrinsics3f& intrinsics,
                        const DepthConverterT& depth_converter, typename DepthConverterT::RawDepth* depth_data,
                        size_t image_w, size_t image_h) {
  b200::cloud_to_depth(points, nullptr, nullptr, intrinsics, depth_converter, nullptr, depth_data, image_w, image_h);
}

template <class DepthConverterT>
void pointsToDepthImage(const ConstVectorSetMatrixMap3f& points, const RigidTransform3f& extrinsics,
                        const b200::Intrinsics3f& intrinsics, const DepthConverterT& depth_converter,
                        typename DepthConverterT::RawDepth* depth_data, size_t image_w, size_t image_h) {
  b200::cloud_to_depth(points, nullptr, &extrinsics, intrinsics, depth_converter, nullptr, depth_data, image_w,
                       image_h);
}

template <class DepthConverterT>
void pointsColorsToRGBDImages(const ConstVectorSetMatrixMap3f& points, const ConstVectorSetMatrixMap3f& colors,
                              const b200::Intrinsics3f& intrinsics, const DepthConverterT& depth_converter,
                              unsigned char* rgb_data, typename DepthConverterT::RawDepth* depth_data, size_t image_w,
                              size_t image_h) {
  b200::cloud_to_depth(points, &colors, nullptr, intrinsics, depth_converter, rgb_data, depth_data, image_w, image_h);
}

template <class DepthConverterT>
void pointsColorsToRGBDImages(const ConstVectorSetMatrixMap3f& points, const ConstVectorSetMatrixMap3f& colors,
                              const RigidTransform3f& extrinsics, const b200::Intrinsics3f& intrinsics,
                              const DepthConverterT& depth_converter, unsigned char* rgb_data,
                              typename DepthConverterT::RawDepth* depth_data, size_t image_w, size_t image_h) {
  b200::cloud_to_depth(points, &colors, &extrinsics, intrinsics, depth_converter, rgb_data, depth_data, image_w,
                       image_h);
}

// IndexT is deduced from the output; PointT (float only) cannot be deduced from the Eigen-free map and defaults to
// float. Empty pixels hold the maximum of IndexT.
template <typename PointT = float, typename IndexT = size_t>
void pointsToIndexMap(const ConstVectorSetMatrixMap3f& points, const b200::Intrinsics3f& intrinsics,
                      IndexT* index_map_data, size_t image_w, size_t image_h) {
  b200::cloud_to_index_map<PointT>(points, nullptr, intrinsics, index_map_data, image_w, image_h);
}

template <typename PointT = float, typename IndexT = size_t>
void pointsToIndexMap(const ConstVectorSetMatrixMap3f& points, const RigidTransform3f& extrinsics,
                      const b200::Intrinsics3f& intrinsics, IndexT* index_map_data, size_t image_w, size_t image_h) {
  b200::cloud_to_index_map<PointT>(points, &extrinsics, intrinsics, index_map_data, image_w, image_h);
}

}  // namespace cilantro
