// Same include path as cilantro's core/principal_component_analysis.hpp; the GPU-native drop-in lives in b200_shims.hpp.
#pragma once
#include "../b200_shims.hpp"
