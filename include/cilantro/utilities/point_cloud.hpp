// Same include path as cilantro's utilities/point_cloud.hpp; the GPU-native drop-in lives in b200_shims.hpp.
#pragma once
#include "../b200_shims.hpp"
#include "../core/image_point_cloud_conversions.hpp"
#include "../core/normal_estimation.hpp"
