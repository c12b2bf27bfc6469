// Same include path as cilantro's registration/icp_common_instances.hpp; the GPU-native drop-ins live in b200_shims.hpp
// and, for SimpleCombinedMetricRigidProjectiveICP3f, in correspondence_search/correspondence_search_projective.hpp.
#pragma once
#include "../b200_shims.hpp"
#include "../correspondence_search/correspondence_search_projective.hpp"
