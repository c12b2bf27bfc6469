// Same include path as cilantro's correspondence_search/common_transformable_feature_adaptors.hpp; the feature adaptors
// (PointFeaturesAdaptor3f ... PointNormalColorFeaturesAdaptor3f) live in b200_shims.hpp.
#pragma once
#include "../b200_shims.hpp"
