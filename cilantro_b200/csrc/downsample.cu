// Voxel-grid downsampling (product code, sm_90a) — §8(f) rank 2.
// Replaces GridAccumulator::build_index_ (core/grid_accumulator.hpp:146-199) + Points[Normals][Colors]
// GridDownsampler::getDownsampled* (core/grid_downsampler.hpp) behind PointCloud::gridDownsample
// (utilities/point_cloud.hpp:246-290).
//
// Reference: bin of a point = floor(p[i] * (1 / bin_size)) per axis (grid_accumulator.hpp:117-126); a
// std::map keyed lexicographically on (x, y, z) (:9-39) accumulates, per bin, the fp32 point sum, the
// sign-consistent normal sum (common_accumulators.hpp:122-131) and the colour sum in point-index order
// (serial build, :187-199), and the output is sum / count per bin with at least min_points_in_bin points
// — in map order for the default parallel build (:177-181), in first-occurrence order for the serial one
// (:194-197). (The parallel build merges per-thread partial sums in arrival order, so its rounding is
// not reproducible; this path reproduces the serial sums bit for bit and offers both output orders.)
//
// Here: (1) bin coordinates -> one 64-bit key, x most significant (the map's order), relative to the
// cloud's minimum bin; (2) stable radix sort of (key, point index) on the bits the key range needs
// (radix_sort.cu) — inside a bin the points stay in index order; (3) head flags + scan -> bin starts;
// (4) one thread per bin replays the reference's sequential accumulation; (5) optional re-ordering of
// the bins by their first point index, compaction by min_points_in_bin, emit.
#include "cb_internal.hpp"
#include "launch.cuh"
#include <algorithm>
#include <cmath>
#include <vector>

using namespace cb;

namespace {

constexpr int kThreads = 256;

struct BinGrid {
  float inv;                // 1 / bin_size (fp32, like bin_size_.cwiseInverse())
  long long mnx, mny, mnz;  // minimum bin coordinate per axis
  uint64_t ny, nz;
  uint64_t none;            // key of a point with a non-finite coordinate: one past the largest bin key
};

// (ptrdiff_t)std::floor(point[i] * bin_size_inv_[i]) relative to the cloud's minimum bin. The bounding box
// covers every finite coordinate, so a finite point's bin lies inside the grid.
__device__ __forceinline__ uint64_t rel_bin(float v, float inv, long long mn) {
  return (uint64_t)(__float2ll_rd(__fmul_rn(v, inv)) - mn);
}

// A point with a NaN / Inf coordinate belongs to no bin (its bin is undefined in the reference): it gets the
// key g.none, sorts after every finite point and is left out of the bins.
__global__ void bin_key_kernel(const float* __restrict__ raw, size_t n, BinGrid g, uint64_t* __restrict__ keys,
                               uint32_t* __restrict__ vals) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float x = raw[3 * i], y = raw[3 * i + 1], z = raw[3 * i + 2];
    uint64_t key = g.none;
    if (isfinite(x) && isfinite(y) && isfinite(z)) {
      const uint64_t ix = rel_bin(x, g.inv, g.mnx), iy = rel_bin(y, g.inv, g.mny), iz = rel_bin(z, g.inv, g.mnz);
      key = (ix * g.ny + iy) * g.nz + iz;
    }
    keys[i] = key;
    vals[i] = (uint32_t)i;
  }
}

__global__ void head_flag_kernel(const uint64_t* __restrict__ keys, size_t n, uint64_t none,
                                 uint32_t* __restrict__ flags) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i <= n; i += (size_t)gridDim.x * blockDim.x)
    flags[i] = (i < n && keys[i] != none && (i == 0 || keys[i] != keys[i - 1])) ? 1u : 0u;
}

// after the exclusive scan, flags[i] = number of bin heads before i and flags[n] = nbins; heads write their
// position, and bin_start[nbins] = the end of the finite points (the first non-finite one, or n)
__global__ void bin_start_kernel(const uint64_t* __restrict__ keys, size_t n, uint64_t none,
                                 const uint32_t* __restrict__ scanned, uint32_t* __restrict__ bin_start) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (i == 0 || keys[i] != keys[i - 1]) bin_start[scanned[i]] = (uint32_t)i;
    if (i == n - 1 && keys[i] != none) bin_start[scanned[n]] = (uint32_t)n;
  }
}

struct BinOut {
  float* pts;    // 3 per bin
  float* nrm;    // 3 per bin or nullptr
  float* col;    // 3 per bin or nullptr
  uint32_t* cnt; // points per bin
  uint32_t* first;  // lowest point index of the bin
};

__global__ void bin_reduce_kernel(const float* __restrict__ raw, const float* __restrict__ raw_nrm,
                                  const float* __restrict__ raw_col, const uint32_t* __restrict__ order,
                                  const uint32_t* __restrict__ bin_start, uint32_t nbins, BinOut o) {
  for (uint32_t b = blockIdx.x * blockDim.x + threadIdx.x; b < nbins; b += gridDim.x * blockDim.x) {
    const uint32_t s = bin_start[b], e = bin_start[b + 1];
    uint32_t i = order[s];
    float px = raw[3 * (size_t)i], py = raw[3 * (size_t)i + 1], pz = raw[3 * (size_t)i + 2];  // buildAccumulator
    float nx = 0.f, ny = 0.f, nz = 0.f, cr = 0.f, cg = 0.f, cb_ = 0.f;
    if (raw_nrm) { nx = raw_nrm[3 * (size_t)i]; ny = raw_nrm[3 * (size_t)i + 1]; nz = raw_nrm[3 * (size_t)i + 2]; }
    if (raw_col) { cr = raw_col[3 * (size_t)i]; cg = raw_col[3 * (size_t)i + 1]; cb_ = raw_col[3 * (size_t)i + 2]; }
    o.first[b] = i;
    for (uint32_t j = s + 1; j < e; j++) {  // addToAccumulator, in point-index order
      i = order[j];
      px = __fadd_rn(px, raw[3 * (size_t)i]);
      py = __fadd_rn(py, raw[3 * (size_t)i + 1]);
      pz = __fadd_rn(pz, raw[3 * (size_t)i + 2]);
      if (raw_nrm) {
        const float ax = raw_nrm[3 * (size_t)i], ay = raw_nrm[3 * (size_t)i + 1], az = raw_nrm[3 * (size_t)i + 2];
        const float d = __fadd_rn(__fmul_rn(nx, ax), __fadd_rn(__fmul_rn(ny, ay), __fmul_rn(nz, az)));
        if (d < 0.f) {
          nx = __fsub_rn(nx, ax); ny = __fsub_rn(ny, ay); nz = __fsub_rn(nz, az);
        } else {
          nx = __fadd_rn(nx, ax); ny = __fadd_rn(ny, ay); nz = __fadd_rn(nz, az);
        }
      }
      if (raw_col) {
        cr = __fadd_rn(cr, raw_col[3 * (size_t)i]);
        cg = __fadd_rn(cg, raw_col[3 * (size_t)i + 1]);
        cb_ = __fadd_rn(cb_, raw_col[3 * (size_t)i + 2]);
      }
    }
    const uint32_t count = e - s;
    const float scale = __fdiv_rn(1.0f, (float)count);  // (ScalarT)(1.0) / pointCount
    o.cnt[b] = count;
    o.pts[3 * (size_t)b] = __fmul_rn(scale, px);
    o.pts[3 * (size_t)b + 1] = __fmul_rn(scale, py);
    o.pts[3 * (size_t)b + 2] = __fmul_rn(scale, pz);
    if (raw_nrm) {  // (scale * normalSum).normalized(): divide by sqrt(squaredNorm) when it is > 0
      const float wx = __fmul_rn(scale, nx), wy = __fmul_rn(scale, ny), wz = __fmul_rn(scale, nz);
      const float z = __fadd_rn(__fmul_rn(wx, wx), __fadd_rn(__fmul_rn(wy, wy), __fmul_rn(wz, wz)));
      if (z > 0.f) {
        const float nn = __fsqrt_rn(z);
        o.nrm[3 * (size_t)b] = __fdiv_rn(wx, nn);
        o.nrm[3 * (size_t)b + 1] = __fdiv_rn(wy, nn);
        o.nrm[3 * (size_t)b + 2] = __fdiv_rn(wz, nn);
      } else {
        o.nrm[3 * (size_t)b] = wx;
        o.nrm[3 * (size_t)b + 1] = wy;
        o.nrm[3 * (size_t)b + 2] = wz;
      }
    }
    if (raw_col) {
      o.col[3 * (size_t)b] = __fmul_rn(scale, cr);
      o.col[3 * (size_t)b + 1] = __fmul_rn(scale, cg);
      o.col[3 * (size_t)b + 2] = __fmul_rn(scale, cb_);
    }
  }
}

__global__ void first_key_kernel(const uint32_t* __restrict__ first, uint32_t nbins, uint64_t* __restrict__ keys,
                                 uint32_t* __restrict__ vals) {
  for (uint32_t b = blockIdx.x * blockDim.x + threadIdx.x; b < nbins; b += gridDim.x * blockDim.x) {
    keys[b] = first[b];
    vals[b] = b;
  }
}

// rank r of the output order -> bin rank_bin[r] (or r itself); valid[r] = count >= min_points
__global__ void valid_flag_kernel(const uint32_t* __restrict__ rank_bin, const uint32_t* __restrict__ cnt,
                                  uint32_t nbins, uint32_t min_points, uint32_t* __restrict__ flags) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r <= nbins; r += gridDim.x * blockDim.x)
    flags[r] = (r < nbins && cnt[rank_bin ? rank_bin[r] : r] >= min_points) ? 1u : 0u;
}

__global__ void emit_kernel(const uint32_t* __restrict__ rank_bin, const uint32_t* __restrict__ scanned, BinOut o,
                            uint32_t nbins, uint32_t min_points, float* __restrict__ out_pts,
                            float* __restrict__ out_nrm, float* __restrict__ out_col) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < nbins; r += gridDim.x * blockDim.x) {
    const uint32_t b = rank_bin ? rank_bin[r] : r;
    if (o.cnt[b] < min_points) continue;
    const size_t d = scanned[r];
#pragma unroll
    for (int c = 0; c < 3; c++) {
      out_pts[3 * d + c] = o.pts[3 * (size_t)b + c];
      if (out_nrm) out_nrm[3 * d + c] = o.nrm[3 * (size_t)b + c];
      if (out_col) out_col[3 * d + c] = o.col[3 * (size_t)b + c];
    }
  }
}

int bits_for(uint64_t count) {  // bits needed to represent values 0 .. count-1
  int b = 0;
  while (b < 64 && (count - 1) >> b) ++b;
  return std::max(b, 1);
}

using DeviceBufs = DeviceScope;  // scoped stream-ordered allocations (cb_internal.hpp)

// Device-side core: inputs are packed xyz arrays in device memory; outputs are device arrays of *out_n entries
// allocated from the caller's scope `out` (nullptr when *out_n == 0).
int downsample_device(cb_context* ctx, DeviceScope& out, const float* d_raw, const float* d_nrm, const float* d_col,
                      size_t n, float bin_size, size_t min_points, int order, float** out_pts, float** out_nrm,
                      float** out_col, size_t* out_n) {
  *out_pts = nullptr;
  if (out_nrm) *out_nrm = nullptr;
  if (out_col) *out_col = nullptr;
  *out_n = 0;
  if (n == 0) return CB_OK;
  CB_CHECK(n < (1ull << 31), CB_ERR_INVALID, "point sets of >= 2^31 points are not supported");
  CB_CHECK(bin_size > 0.f && std::isfinite(bin_size), CB_ERR_INVALID, "bin_size must be positive and finite");
  float mn[3], mx[3];
  CB_TRY(points_bbox(ctx, d_raw, n, mn, mx));
  BinGrid g;
  g.inv = 1.0f / bin_size;
  long long lo[3];
  uint64_t dim[3];
  for (int a = 0; a < 3; a++) {
    const float flo = std::floor(mn[a] * g.inv), fhi = std::floor(mx[a] * g.inv);
    CB_CHECK(std::fabs(flo) < 4.0e18f && std::fabs(fhi) < 4.0e18f, CB_ERR_UNSUPPORTED,
             "bin coordinates exceed 64 bits (bin_size too small for the coordinates)");
    lo[a] = (long long)flo;
    dim[a] = (uint64_t)((long long)fhi - lo[a]) + 1u;
  }
  const long double total = (long double)dim[0] * (long double)dim[1] * (long double)dim[2];
  CB_CHECK(total < 9.0e18L, CB_ERR_UNSUPPORTED, "bin grid too large for a 64-bit key (bin_size too small for the extent)");
  g.mnx = lo[0]; g.mny = lo[1]; g.mnz = lo[2];
  g.ny = dim[1]; g.nz = dim[2];
  g.none = dim[0] * dim[1] * dim[2];
  const int key_bits = bits_for(g.none + 1);

  DeviceBufs bufs(ctx);
  uint64_t *d_keys, *d_keys2;
  uint32_t *d_vals, *d_vals2, *d_flags, *d_start;
  CB_TRY(bufs.alloc(&d_keys, n));
  CB_TRY(bufs.alloc(&d_keys2, n));
  CB_TRY(bufs.alloc(&d_vals, n));
  CB_TRY(bufs.alloc(&d_vals2, n));
  CB_TRY(bufs.alloc(&d_flags, n + 2));
  const int nb = grid_for(ctx, n, kThreads, 16);
  CB_TRY(launch(ctx, bin_key_kernel, nb, kThreads, 0, d_raw, n, g, d_keys, d_vals));
  CB_TRY(radix_sort_pairs_u64(ctx, d_keys, d_vals, d_keys2, d_vals2, n, key_bits));
  CB_TRY(launch(ctx, head_flag_kernel, nb, kThreads, 0, d_keys, n, g.none, d_flags));
  CB_TRY(exclusive_scan_u32(ctx, d_flags, n + 1, 0u));  // flags[n] = number of bins; flags[n + 1] = sentinel
  uint32_t nbins = 0;
  CB_CUDA(cudaMemcpyAsync(&nbins, d_flags + n, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  CB_CHECK(nbins <= n, CB_ERR_CUDA, "internal: inconsistent bin count");
  if (nbins == 0) return CB_OK;  // no point with three finite coordinates
  CB_TRY(bufs.alloc(&d_start, (size_t)nbins + 1));
  CB_TRY(launch(ctx, bin_start_kernel, nb, kThreads, 0, d_keys, n, g.none, d_flags, d_start));
  BinOut o;
  o.nrm = nullptr;
  o.col = nullptr;
  CB_TRY(bufs.alloc(&o.pts, 3 * (size_t)nbins));
  if (d_nrm) CB_TRY(bufs.alloc(&o.nrm, 3 * (size_t)nbins));
  if (d_col) CB_TRY(bufs.alloc(&o.col, 3 * (size_t)nbins));
  CB_TRY(bufs.alloc(&o.cnt, nbins));
  CB_TRY(bufs.alloc(&o.first, nbins));
  const int bb = grid_for(ctx, nbins, kThreads, 16);
  CB_TRY(launch(ctx, bin_reduce_kernel, bb, kThreads, 0, d_raw, d_nrm, d_col, d_vals, d_start, nbins, o));
  // output order
  uint32_t* d_rank_bin = nullptr;
  if (order == 1 && nbins > 1) {  // first-occurrence order (serial build): sort the bins by their first index
    CB_TRY(launch(ctx, first_key_kernel, bb, kThreads, 0, o.first, nbins, d_keys, d_vals));
    CB_TRY(radix_sort_pairs_u64(ctx, d_keys, d_vals, d_keys2, d_vals2, nbins, bits_for(n)));
    d_rank_bin = d_vals;
  }
  size_t m = nbins;
  const uint32_t minp = (uint32_t)std::min<size_t>(min_points, 0xffffffffu);
  CB_TRY(launch(ctx, valid_flag_kernel, bb, kThreads, 0, d_rank_bin, o.cnt, nbins, minp, d_flags));
  CB_TRY(exclusive_scan_u32(ctx, d_flags, (size_t)nbins + 1, 0u));
  if (minp > 1) {
    uint32_t mm = 0;
    CB_CUDA(cudaMemcpyAsync(&mm, d_flags + nbins, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    m = mm;
  }
  *out_n = m;
  if (m == 0) return CB_OK;
  float *r_pts = nullptr, *r_nrm = nullptr, *r_col = nullptr;
  CB_TRY(out.alloc(&r_pts, 3 * m));
  if (d_nrm && out_nrm) CB_TRY(out.alloc(&r_nrm, 3 * m));
  if (d_col && out_col) CB_TRY(out.alloc(&r_col, 3 * m));
  CB_TRY(launch(ctx, emit_kernel, bb, kThreads, 0, d_rank_bin, d_flags, o, nbins, minp, r_pts, r_nrm, r_col));
  *out_pts = r_pts;
  if (r_nrm) *out_nrm = r_nrm;
  if (r_col) *out_col = r_col;
  return CB_OK;
}

}  // namespace

extern "C" int cb_grid_downsample(cb_context* ctx, const float* xyz, const float* normals, const float* colors,
                                  size_t n, float bin_size, size_t min_points_in_bin, int order, float* out_xyz,
                                  float* out_normals, float* out_colors, size_t* out_n) {
  CB_CHECK(ctx && out_n && (n == 0 || (xyz && out_xyz)), CB_ERR_INVALID, "null argument");
  CB_CHECK(order == 0 || order == 1, CB_ERR_INVALID, "order must be 0 (bin order) or 1 (first occurrence)");
  CB_CHECK(!normals || out_normals, CB_ERR_INVALID, "normals given but out_normals is null");
  CB_CHECK(!colors || out_colors, CB_ERR_INVALID, "colors given but out_colors is null");
  CB_CUDA(cudaSetDevice(ctx->device));
  *out_n = 0;
  if (n == 0) return CB_OK;
  DeviceBufs in(ctx);
  float *d_raw, *d_nrm = nullptr, *d_col = nullptr;
  CB_TRY(in.alloc(&d_raw, 3 * n));
  CB_CUDA(cudaMemcpyAsync(d_raw, xyz, 3 * n * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  if (normals) {
    CB_TRY(in.alloc(&d_nrm, 3 * n));
    CB_CUDA(cudaMemcpyAsync(d_nrm, normals, 3 * n * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  }
  if (colors) {
    CB_TRY(in.alloc(&d_col, 3 * n));
    CB_CUDA(cudaMemcpyAsync(d_col, colors, 3 * n * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  }
  float *o_pts = nullptr, *o_nrm = nullptr, *o_col = nullptr;
  size_t m = 0;
  CB_TRY(downsample_device(ctx, in, d_raw, d_nrm, d_col, n, bin_size, min_points_in_bin, order, &o_pts, &o_nrm, &o_col,
                           &m));
  if (m > 0) {
    CB_CUDA(cudaMemcpyAsync(out_xyz, o_pts, 3 * m * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    if (o_nrm) CB_CUDA(cudaMemcpyAsync(out_normals, o_nrm, 3 * m * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    if (o_col) CB_CUDA(cudaMemcpyAsync(out_colors, o_col, 3 * m * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  }
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  *out_n = m;
  return CB_OK;
}

extern "C" int cb_cloud_grid_downsample(cb_context* ctx, const cb_cloud* cloud, float bin_size,
                                        size_t min_points_in_bin, int order, cb_cloud** out, float* gpu_ms) {
  CB_CHECK(ctx && cloud && out, CB_ERR_INVALID, "null argument");
  CB_CHECK(cloud->ctx == ctx, CB_ERR_INVALID, "cloud belongs to another context");
  CB_CHECK(order == 0 || order == 1, CB_ERR_INVALID, "order must be 0 (bin order) or 1 (first occurrence)");
  CB_CUDA(cudaSetDevice(ctx->device));
  *out = nullptr;
  ScopedEvents ev;
  if (gpu_ms) {
    *gpu_ms = 0.f;
    CB_TRY(ev.create());
    CB_CUDA(cudaEventRecord(ev.e0, ctx->stream));
  }
  DeviceBufs bufs(ctx);
  float *o_pts = nullptr, *o_nrm = nullptr;
  size_t m = 0;
  CB_TRY(downsample_device(ctx, bufs, cloud->d_raw, cloud->d_raw_nrm, nullptr, cloud->n, bin_size, min_points_in_bin, order,
                           &o_pts, &o_nrm, nullptr, &m));
  if (gpu_ms) CB_CUDA(cudaEventRecord(ev.e1, ctx->stream));
  CB_TRY(cb_cloud_create_from_device(ctx, o_pts, o_nrm, m, cloud->index_offset, out));
  if (gpu_ms) {
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    CB_CUDA(cudaEventElapsedTime(gpu_ms, ev.e0, ev.e1));
  }
  return CB_OK;
}

extern "C" int cb_cloud_download(cb_context* ctx, const cb_cloud* cloud, float* xyz, float* normals) {
  CB_CHECK(ctx && cloud, CB_ERR_INVALID, "null argument");
  CB_CHECK(cloud->ctx == ctx, CB_ERR_INVALID, "cloud belongs to another context");
  CB_CHECK(!normals || cloud->d_raw_nrm || cloud->n == 0, CB_ERR_INVALID, "cloud has no normals");
  CB_CUDA(cudaSetDevice(ctx->device));
  if (cloud->n == 0) return CB_OK;
  if (xyz) CB_CUDA(cudaMemcpyAsync(xyz, cloud->d_raw, 3 * cloud->n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  if (normals)
    CB_CUDA(cudaMemcpyAsync(normals, cloud->d_raw_nrm, 3 * cloud->n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  return CB_OK;
}
