#pragma once
#include "cb_internal.hpp"

namespace cb {

constexpr int kMomentValues = 10;

// Launches the moments kernel over d_raw (packed xyz, n points) with the given shift; the reduced
// values land in ctx->d_result[0..9] (stream-ordered). finite_only: skip points with a NaN / Inf
// coordinate (result[0] is then the number of finite points).
int launch_moments(cb_context* ctx, const float* d_raw, size_t n, const float* shift3, bool finite_only = false);

// Reads ctx->d_result[0..count) back to the host (after an optional cross-rank all-reduce).
int fetch_result(cb_context* ctx, int count, bool allreduce, double* out);

}  // namespace cb
