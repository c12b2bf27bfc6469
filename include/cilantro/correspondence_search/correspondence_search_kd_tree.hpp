// Same include path as cilantro's correspondence_search/correspondence_search_kd_tree.hpp; the GPU-native drop-in lives in b200_shims.hpp.
#pragma once
#include "../b200_shims.hpp"
