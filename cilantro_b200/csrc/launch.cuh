// Kernel launches of libcilantro_b200.so. Every launch of the library goes through these functions: each one is on the
// context's stream, is counted in cb_context::launches (the kernel_launches of every result) and has its launch error
// checked at once, so a failed launch is reported by the call that made it.
#pragma once
#include <algorithm>
#include <cstring>
#include <utility>
#include "cb_internal.hpp"

namespace cb {

// Blocks of a grid-stride launch over `work` items, `per_block` items per block: enough blocks to cover the work, at
// most per_sm blocks per SM, at least one.
inline int grid_for(const cb_context* ctx, size_t work, size_t per_block, int per_sm = 8) {
  return (int)std::max<size_t>(1, std::min<size_t>((size_t)ctx->sm_count * per_sm, (work + per_block - 1) / per_block));
}

// Counts one launch whose enqueue returned `e`.
inline int launched(cb_context* ctx, cudaError_t e) {
  ctx->launches += 1;
  CB_CUDA(e);
  return CB_OK;
}

// kernel<<<grid, block, smem, ctx->stream>>>(args...)
template <class... Params, class... Args>
int launch(cb_context* ctx, void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, Args&&... args) {
  kernel<<<grid, block, smem, ctx->stream>>>(std::forward<Args>(args)...);
  return launched(ctx, cudaGetLastError());
}

// The same with programmatic stream serialization (programmatic dependent launch, sm_90+): the kernel may be scheduled
// while the previous kernel on the stream is still running, so it must wait (griddepcontrol.wait) before it touches
// anything that kernel wrote.
template <class... Params, class... Args>
int launch_pdl(cb_context* ctx, void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, Args&&... args) {
  cudaLaunchConfig_t cfg;
  std::memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = ctx->stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return launched(ctx, cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...));
}

// A cooperative launch (every block resident at once, grid-wide synchronisation allowed); args as for
// cudaLaunchCooperativeKernel.
inline int launch_cooperative(cb_context* ctx, const void* kernel, dim3 grid, dim3 block, void** args) {
  return launched(ctx, cudaLaunchCooperativeKernel(kernel, grid, block, args, 0, ctx->stream));
}

}  // namespace cb
