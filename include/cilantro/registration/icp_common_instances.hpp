// Same include path as cilantro's registration/icp_common_instances.hpp; the GPU-native drop-in lives in b200_shims.hpp.
#pragma once
#include "../b200_shims.hpp"
