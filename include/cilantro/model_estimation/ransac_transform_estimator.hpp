// Same include path as cilantro's model_estimation/ransac_transform_estimator.hpp; the GPU-native drop-in lives in b200_shims.hpp.
#pragma once
#include "../b200_shims.hpp"
