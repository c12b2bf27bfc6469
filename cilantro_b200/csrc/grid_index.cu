// Uniform-grid index build (product code, sm_90a). One-time per cloud; the GPU counterpart of the
// reference's single-threaded kd-tree build (core/kd_tree.hpp:162-170 ->
// 3rd_party/nanoflann/nanoflann.hpp:1661-1687 buildIndex / :1150-1212 divideTree).
//
// Pipeline (all on the context stream):
//   bbox reduce -> [host: pick cell edge] -> cell id + histogram -> occupancy stats
//   (-> shrink the cell edge and redo while non-empty cells hold too many points)
//   -> exclusive scan -> atomic scatter of point indices -> per-cell index sort (or, when some cell
//   holds more than kHugeCell points, one stable radix sort of (cell, index)) -> gather into the
//   cell-sorted float4 arrays. Either way every cell lists its points in ascending original index.
#include "cb_internal.hpp"
#include "nn_search.cuh"
#include <cfloat>
#include <cmath>
#include <algorithm>

namespace cb {

namespace {

constexpr int kThreads = 256;
constexpr int kMaxDim = 1024;        // cells per axis (bounds the cell_coord rounding error, nn_search.cuh)
constexpr double kTargetOcc = 2.0;   // points per non-empty cell aimed for

__device__ __forceinline__ int float_to_ordered(float f) {
  int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7fffffff;
}
__host__ __device__ __forceinline__ float ordered_to_float(int i) {
  int j = i >= 0 ? i : i ^ 0x7fffffff;
#ifdef __CUDA_ARCH__
  return __int_as_float(j);
#else
  float f;
  memcpy(&f, &j, 4);
  return f;
#endif
}

__global__ void bbox_init_kernel(int* bb) {
  if (threadIdx.x < 3) bb[threadIdx.x] = 0x7fffffff;        // mins
  else if (threadIdx.x < 6) bb[threadIdx.x] = (int)0x80000000;  // maxs
}

__global__ void bbox_kernel(const float* __restrict__ raw, size_t n, int* bb) {
  float mn[3] = {3.0e38f, 3.0e38f, 3.0e38f}, mx[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
#pragma unroll
    for (int a = 0; a < 3; a++) {
      float v = raw[3 * i + a];
      if (v == v && fabsf(v) < 3.0e38f) {  // ignore NaN / Inf coordinates for the extent
        mn[a] = fminf(mn[a], v);
        mx[a] = fmaxf(mx[a], v);
      }
    }
  }
#pragma unroll
  for (int a = 0; a < 3; a++) {
    for (int o = 16; o > 0; o >>= 1) {
      mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
      mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
    }
  }
  // warp results -> shared memory -> 6 atomics per block (one per warp was ~60 k contended atomics at 1 M)
  __shared__ float s_mn[kThreads / 32][3], s_mx[kThreads / 32][3];
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int a = 0; a < 3; a++) {
      s_mn[threadIdx.x >> 5][a] = mn[a];
      s_mx[threadIdx.x >> 5][a] = mx[a];
    }
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    float lo = s_mn[0][threadIdx.x], hi = s_mx[0][threadIdx.x];
    for (int w = 1; w < (int)(blockDim.x >> 5); w++) {
      lo = fminf(lo, s_mn[w][threadIdx.x]);
      hi = fmaxf(hi, s_mx[w][threadIdx.x]);
    }
    atomicMin(bb + threadIdx.x, float_to_ordered(lo));
    atomicMax(bb + 3 + threadIdx.x, float_to_ordered(hi));
  }
}

struct GridParams {
  float ox, oy, oz, inv_h;
  int nx, ny, nz;
};

__device__ __forceinline__ uint32_t cell_of(const GridParams& g, float x, float y, float z) {
  int cx = (int)floorf(cell_coord(x, g.ox, g.inv_h));
  int cy = (int)floorf(cell_coord(y, g.oy, g.inv_h));
  int cz = (int)floorf(cell_coord(z, g.oz, g.inv_h));
  cx = min(max(cx, 0), g.nx - 1);
  cy = min(max(cy, 0), g.ny - 1);
  cz = min(max(cz, 0), g.nz - 1);
  return ((uint32_t)cz * (uint32_t)g.ny + (uint32_t)cy) * (uint32_t)g.nx + (uint32_t)cx;
}

__global__ void hist_kernel(const float* __restrict__ raw, size_t n, GridParams g, uint32_t* __restrict__ cell_id,
                            uint32_t* __restrict__ hist) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t c = cell_of(g, raw[3 * i], raw[3 * i + 1], raw[3 * i + 2]);
    cell_id[i] = c;
    atomicAdd(hist + c, 1u);
  }
}

// stats[0] = number of non-empty cells, stats[1] = max cell count
__global__ void occupancy_kernel(const uint32_t* __restrict__ hist, size_t ncells, unsigned long long* stats) {
  unsigned long long nz = 0;
  unsigned int mx = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < ncells; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t h = hist[i];
    nz += (h != 0);
    mx = max(mx, h);
  }
  for (int o = 16; o > 0; o >>= 1) {
    nz += __shfl_xor_sync(0xffffffffu, nz, o);
    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(stats, nz);
    atomicMax(stats + 1, (unsigned long long)mx);
  }
}

// ---- exclusive scan over uint32 (three phases) -------------------------------------------------
constexpr int kScanItems = 16;
constexpr int kScanBlock = kThreads * kScanItems;  // 4096 elements per block

__global__ void scan_block_kernel(uint32_t* __restrict__ data, size_t n, uint32_t* __restrict__ block_sums) {
  __shared__ uint32_t warp_sums[kThreads / 32];
  const size_t base = (size_t)blockIdx.x * kScanBlock + (size_t)threadIdx.x * kScanItems;
  uint32_t v[kScanItems];
  uint32_t s = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; k++) {
    v[k] = (base + k < n) ? data[base + k] : 0u;
    s += v[k];
  }
  // inclusive scan of per-thread sums within the warp
  uint32_t incl = s;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = (lane < kThreads / 32) ? warp_sums[lane] : 0u;
    uint32_t wi = w;
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += t;
    }
    if (lane < kThreads / 32) warp_sums[lane] = wi - w;  // exclusive
    if (lane == kThreads / 32 - 1) block_sums[blockIdx.x] = wi;
  }
  __syncthreads();
  uint32_t run = warp_sums[warp] + (incl - s);
#pragma unroll
  for (int k = 0; k < kScanItems; k++) {
    if (base + k < n) data[base + k] = run;
    run += v[k];
  }
}

__global__ void scan_sums_kernel(uint32_t* __restrict__ block_sums, size_t nblocks) {
  // single block; serial over chunks of blockDim with a running carry
  __shared__ uint32_t warp_sums[32];
  __shared__ uint32_t carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (size_t base = 0; base < nblocks; base += blockDim.x) {
    size_t i = base + threadIdx.x;
    uint32_t v = (i < nblocks) ? block_sums[i] : 0u;
    uint32_t incl = v;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      uint32_t w = (lane < (int)(blockDim.x >> 5)) ? warp_sums[lane] : 0u;
      uint32_t wi = w;
      for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) wi += t;
      }
      warp_sums[lane] = wi - w;
    }
    __syncthreads();
    uint32_t carry = carry_s;
    uint32_t excl = carry + warp_sums[warp] + (incl - v);
    if (i < nblocks) block_sums[i] = excl;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry_s = excl + v;
    __syncthreads();
  }
}

__global__ void scan_add_kernel(uint32_t* __restrict__ data, size_t n, const uint32_t* __restrict__ block_sums,
                                uint32_t total_n) {
  const size_t base = (size_t)blockIdx.x * kScanBlock;
  const uint32_t off = block_sums[blockIdx.x];
  for (int k = threadIdx.x; k < kScanBlock; k += blockDim.x) {
    size_t i = base + k;
    if (i < n) data[i] += off;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) data[n] = total_n;  // sentinel cell_start[ncells] = n
}

__global__ void scatter_kernel(const uint32_t* __restrict__ cell_id, size_t n, const uint32_t* __restrict__ cell_start,
                               uint32_t* __restrict__ cursor, uint32_t* __restrict__ perm) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t c = cell_id[i];
    uint32_t pos = cell_start[c] + atomicAdd(cursor + c, 1u);
    perm[pos] = (uint32_t)i;
  }
}

// Make the layout independent of atomic arrival order: sort each cell's indices ascending.
// Small cells: one thread per cell, insertion sort. Cells above kBigCell are left to
// sort_big_cells_kernel (rank sort by one block per cell, O(m^2) for m points). A grid with a cell
// above kHugeCell (degenerate inputs: millions of coincident points, a scan collapsed into a few cells
// by a far outlier) skips all three kernels and is laid out by a stable radix sort instead
// (ensure_index).
constexpr uint32_t kBigCell = 32;
constexpr uint32_t kHugeCell = 1u << 16;

__global__ void sort_small_cells_kernel(const uint32_t* __restrict__ cell_start, size_t ncells,
                                        uint32_t* __restrict__ perm, uint32_t* __restrict__ big_list,
                                        uint32_t* __restrict__ big_count) {
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < ncells; c += (size_t)gridDim.x * blockDim.x) {
    const uint32_t b = cell_start[c], e = cell_start[c + 1];
    const uint32_t m = e - b;
    if (m < 2) continue;
    if (m > kBigCell) {
      uint32_t slot = atomicAdd(big_count, 1u);
      big_list[slot] = (uint32_t)c;
      continue;
    }
    for (uint32_t i = b + 1; i < e; ++i) {
      uint32_t v = perm[i];
      uint32_t j = i;
      while (j > b && perm[j - 1] > v) {
        perm[j] = perm[j - 1];
        --j;
      }
      perm[j] = v;
    }
  }
}

__global__ void sort_big_cells_kernel(const uint32_t* __restrict__ cell_start, const uint32_t* __restrict__ big_list,
                                      const uint32_t* __restrict__ big_count, uint32_t* __restrict__ perm,
                                      uint32_t* __restrict__ tmp) {
  for (uint32_t k = blockIdx.x; k < *big_count; k += gridDim.x) {
    const uint32_t c = big_list[k];
    const uint32_t b = cell_start[c], e = cell_start[c + 1];
    for (uint32_t i = b + threadIdx.x; i < e; i += blockDim.x) tmp[i] = perm[i];
    __syncthreads();
    for (uint32_t i = b + threadIdx.x; i < e; i += blockDim.x) {
      const uint32_t v = tmp[i];
      uint32_t rank = 0;
      for (uint32_t j = b; j < e; ++j) rank += (tmp[j] < v);  // indices are distinct
      perm[b + rank] = v;
    }
    __syncthreads();
  }
}

// keys of the stable (cell, index) sort: the radix sort keeps equal cells in input (= index) order
__global__ void cell_keys_kernel(const uint32_t* __restrict__ cell_id, size_t n, uint64_t* __restrict__ keys,
                                 uint32_t* __restrict__ perm) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    keys[i] = cell_id[i];
    perm[i] = (uint32_t)i;
  }
}

__global__ void gather_kernel(const float* __restrict__ raw, const float* __restrict__ raw_nrm,
                              const uint32_t* __restrict__ perm, size_t n, float4* __restrict__ pts,
                              float4* __restrict__ nrm) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const uint32_t s = perm[i];
    pts[i] = make_float4(raw[3 * (size_t)s], raw[3 * (size_t)s + 1], raw[3 * (size_t)s + 2], __int_as_float((int)s));
    if (nrm) nrm[i] = make_float4(raw_nrm[3 * (size_t)s], raw_nrm[3 * (size_t)s + 1], raw_nrm[3 * (size_t)s + 2], 0.f);
  }
}

// points per coarse block (kBlockCells^3 cells): 64 row ranges of the final cell_start table
__global__ void block_count_kernel(const uint32_t* __restrict__ cell_start, int nx, int ny, int nz, int bx, int by,
                                   int bz, uint32_t* __restrict__ cnt, uint32_t* __restrict__ flag) {
  // one warp per coarse block: lane l takes rows l and l + 32 of the block's 8 x 8 (y, z) rows
  const size_t nb = (size_t)bx * by * bz;
  const int lane = threadIdx.x & 31;
  const size_t warps = ((size_t)gridDim.x * blockDim.x) >> 5;
  for (size_t b = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5; b <= nb; b += warps) {
    if (b == nb) {
      if (lane == 0) flag[b] = 0u;
      continue;
    }
    const int X = (int)(b % bx), Y = (int)((b / bx) % by), Z = (int)(b / ((size_t)bx * by));
    const int x0 = X * kBlockCells, x1 = min(x0 + kBlockCells, nx);
    uint32_t c = 0;
#pragma unroll
    for (int r = lane; r < kBlockCells * kBlockCells; r += 32) {
      const int y = Y * kBlockCells + (r % kBlockCells), z = Z * kBlockCells + (r / kBlockCells);
      if (y < ny && z < nz) {
        const size_t base = ((size_t)z * ny + y) * nx;
        c += cell_start[base + x1] - cell_start[base + x0];
      }
    }
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) {
      cnt[b] = c;
      flag[b] = c > 0 ? 1u : 0u;
    }
  }
}

__global__ void block_emit_kernel(const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ scanned, int bx,
                                  int by, int bz, uint4* __restrict__ blocks) {
  const size_t nb = (size_t)bx * by * bz;
  for (size_t b = blockIdx.x * (size_t)blockDim.x + threadIdx.x; b < nb; b += (size_t)gridDim.x * blockDim.x) {
    if (cnt[b] == 0) continue;
    blocks[scanned[b]] = make_uint4((unsigned)(b % bx), (unsigned)((b / bx) % by), (unsigned)(b / ((size_t)bx * by)), cnt[b]);
  }
}

inline int grid_blocks(const cb_context* ctx, size_t n, int per_sm = 8) {
  size_t want = (n + kThreads - 1) / kThreads;
  size_t cap = (size_t)ctx->sm_count * per_sm;
  return (int)std::max<size_t>(1, std::min(want, cap));
}

}  // namespace

int exclusive_scan_u32(cb_context* ctx, uint32_t* d_data, size_t n, uint32_t total) {
  // d_data has n + 1 entries; on return d_data[i] = sum_{j<i} in[j], d_data[n] = total
  const size_t nblocks = (n + kScanBlock - 1) / kScanBlock;
  DeviceScope scope(ctx);
  uint32_t* d_sums = nullptr;
  CB_TRY(scope.alloc(&d_sums, nblocks));
  scan_block_kernel<<<(unsigned)nblocks, kThreads, 0, ctx->stream>>>(d_data, n, d_sums);
  scan_sums_kernel<<<1, 1024, 0, ctx->stream>>>(d_sums, nblocks);
  scan_add_kernel<<<(unsigned)nblocks, kThreads, 0, ctx->stream>>>(d_data, n, d_sums, total);
  ctx->launches += 3;
  CB_CUDA(cudaGetLastError());
  return CB_OK;
}

int points_bbox(cb_context* ctx, const float* d_raw, size_t n, float mn[3], float mx[3]) {
  DeviceScope scope(ctx);
  int* d_bb = nullptr;
  CB_TRY(scope.alloc(&d_bb, 6));
  bbox_init_kernel<<<1, 32, 0, ctx->stream>>>(d_bb);
  bbox_kernel<<<grid_blocks(ctx, n), kThreads, 0, ctx->stream>>>(d_raw, n, d_bb);
  ctx->launches += 2;
  int h_bb[6];
  CB_CUDA(cudaMemcpyAsync(h_bb, d_bb, sizeof(h_bb), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  for (int a = 0; a < 3; a++) {
    mn[a] = ordered_to_float(h_bb[a]);
    mx[a] = ordered_to_float(h_bb[3 + a]);
    if (!(mn[a] <= mx[a])) mn[a] = mx[a] = 0.f;  // no finite coordinate on this axis
  }
  return CB_OK;
}

int ensure_index(cb_cloud* c) {
  if (c->indexed) return CB_OK;
  cb_context* ctx = c->ctx;
  const size_t n = c->n;
  CB_CHECK(n < (1ull << 31), CB_ERR_INVALID, "point sets of >= 2^31 points are not supported");
  CB_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) {
    c->nx = c->ny = c->nz = 1;
    c->h = c->inv_h = 1.f;
    CB_TRY(c->mem.alloc(&c->d_cell_start, 2));
    CB_CUDA(cudaMemsetAsync(c->d_cell_start, 0, 2 * sizeof(uint32_t), ctx->stream));
    c->indexed = true;
    return CB_OK;
  }
  // 1. bounding box
  float mn[3], mx[3];
  CB_TRY(points_bbox(ctx, c->d_raw, n, mn, mx));
  double ext[3] = {(double)mx[0] - mn[0], (double)mx[1] - mn[1], (double)mx[2] - mn[2]};
  const double max_ext = std::max({ext[0], ext[1], ext[2], 1e-30});

  // 2. cell edge: start from a cube-root density guess, then shrink while the non-empty cells are
  //    over-full (surface-like clouds fill few cells).
  const size_t cell_cap = std::min<size_t>((size_t)1 << 28, std::max<size_t>((size_t)1 << 20, 16 * n));
  double m0 = std::ceil(std::cbrt((double)n / kTargetOcc));
  m0 = std::min<double>(std::max(m0, 1.0), kMaxDim);
  double h = max_ext / m0;

  // Scratch in `scope`; the index arrays in c->mem, so a failure leaves the cloud as it was (not indexed,
  // nothing allocated: every buffer of a failed attempt is freed with its scope or the cloud).
  DeviceScope scope(ctx);
  uint32_t* d_cell_id = nullptr;
  uint32_t* d_hist = nullptr;  // becomes the cell_start of the index
  unsigned long long* d_stats = nullptr;
  CB_TRY(scope.alloc(&d_cell_id, n));
  CB_TRY(scope.alloc(&d_stats, 2));
  GridParams gp;
  size_t ncells = 0;
  double mean_occ = 0;
  unsigned long long max_occ = 0;  // largest cell of the grid in gp
  for (int attempt = 0; attempt < 6; ++attempt) {
    // dims from the edge; keep every axis <= kMaxDim and the table <= cell_cap
    int dims[3];
    for (;;) {
      size_t tot = 1;
      bool ok = true;
      for (int a = 0; a < 3; a++) {
        // one empty margin cell on each side: queries up to a cell outside the bounding box (every
        // ICP run has them along the faces) stay on the pooled "inside the grid" search path
        double d = std::floor(ext[a] / h) + 3.0;
        if (d > kMaxDim) ok = false;
        dims[a] = (int)std::min<double>(d, kMaxDim);
        tot *= (size_t)dims[a];
      }
      if (ok && tot <= cell_cap) break;
      h *= 1.26;
    }
    gp.ox = (float)((double)mn[0] - h);
    gp.oy = (float)((double)mn[1] - h);
    gp.oz = (float)((double)mn[2] - h);
    gp.inv_h = (float)(1.0 / h);
    gp.nx = dims[0];
    gp.ny = dims[1];
    gp.nz = dims[2];
    ncells = (size_t)dims[0] * dims[1] * dims[2];
    CB_TRY(scope.free(d_hist));
    CB_TRY(scope.alloc(&d_hist, ncells + 1));
    CB_CUDA(cudaMemsetAsync(d_hist, 0, (ncells + 1) * sizeof(uint32_t), ctx->stream));
    CB_CUDA(cudaMemsetAsync(d_stats, 0, 2 * sizeof(unsigned long long), ctx->stream));
    hist_kernel<<<grid_blocks(ctx, n), kThreads, 0, ctx->stream>>>(c->d_raw, n, gp, d_cell_id, d_hist);
    occupancy_kernel<<<grid_blocks(ctx, ncells), kThreads, 0, ctx->stream>>>(d_hist, ncells, d_stats);
    ctx->launches += 2;
    unsigned long long h_stats[2];
    CB_CUDA(cudaMemcpyAsync(h_stats, d_stats, sizeof(h_stats), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    mean_occ = (double)n / (double)std::max<unsigned long long>(1, h_stats[0]);
    max_occ = h_stats[1];
    const int maxdim = std::max({dims[0], dims[1], dims[2]});
    if (mean_occ <= 2.0 * kTargetOcc || maxdim >= kMaxDim || ncells * 4 > cell_cap) break;
    // shrink: occupancy of a surface scales ~h^2, of a volume ~h^3; use the square-root (stronger) step
    double f = std::sqrt(mean_occ / kTargetOcc);
    f = std::min(f, 4.0);
    double hn = h / f;
    // never let the finest axis exceed kMaxDim
    hn = std::max(hn, max_ext / (double)(kMaxDim - 1));
    if (hn >= h * 0.95) break;
    h = hn;
  }
  c->ox = gp.ox;
  c->oy = gp.oy;
  c->oz = gp.oz;
  c->inv_h = gp.inv_h;
  c->h = (float)h;
  c->nx = gp.nx;
  c->ny = gp.ny;
  c->nz = gp.nz;
  c->mean_occ = mean_occ;

  // 3. cell_start = exclusive scan of the histogram (in place; d_hist becomes cell_start)
  CB_TRY(exclusive_scan_u32(ctx, d_hist, ncells, (uint32_t)n));
  // 4. point indices in cell order, ascending inside every cell (sums over a cloud in cell order are then the
  //    same on every build)
  uint32_t* d_perm = nullptr;
  CB_TRY(scope.alloc(&d_perm, n));
  if (max_occ <= kHugeCell) {
    uint32_t* d_cursor = nullptr;
    uint32_t* d_big = nullptr;
    uint32_t* d_tmp = nullptr;
    CB_TRY(scope.alloc(&d_cursor, ncells));
    CB_CUDA(cudaMemsetAsync(d_cursor, 0, ncells * sizeof(uint32_t), ctx->stream));
    const size_t big_cap = n / kBigCell + 2;
    CB_TRY(scope.alloc(&d_big, big_cap + 1));
    CB_CUDA(cudaMemsetAsync(d_big, 0, sizeof(uint32_t), ctx->stream));
    CB_TRY(scope.alloc(&d_tmp, n));
    scatter_kernel<<<grid_blocks(ctx, n), kThreads, 0, ctx->stream>>>(d_cell_id, n, d_hist, d_cursor, d_perm);
    sort_small_cells_kernel<<<grid_blocks(ctx, ncells), kThreads, 0, ctx->stream>>>(d_hist, ncells, d_perm,
                                                                                   d_big + 1, d_big);
    sort_big_cells_kernel<<<ctx->sm_count * 2, kThreads, 0, ctx->stream>>>(d_hist, d_big + 1, d_big, d_perm, d_tmp);
    ctx->launches += 3;
  } else {
    // a rank sort of a cell this large would cost O(m^2): sort (cell, index) pairs of the whole cloud instead
    uint64_t* d_keys = nullptr;
    uint64_t* d_keys_tmp = nullptr;
    uint32_t* d_vals_tmp = nullptr;
    CB_TRY(scope.alloc(&d_keys, n));
    CB_TRY(scope.alloc(&d_keys_tmp, n));
    CB_TRY(scope.alloc(&d_vals_tmp, n));
    cell_keys_kernel<<<grid_blocks(ctx, n), kThreads, 0, ctx->stream>>>(d_cell_id, n, d_keys, d_perm);
    ctx->launches += 1;
    int bits = 1;
    while (bits < 32 && ((ncells - 1) >> bits) != 0) ++bits;
    CB_TRY(radix_sort_pairs_u64(ctx, d_keys, d_perm, d_keys_tmp, d_vals_tmp, n, bits));
  }
  // 5. gather
  float4 *d_pts = nullptr, *d_nrm = nullptr;
  CB_TRY(scope.alloc(&d_pts, n));
  if (c->d_raw_nrm) CB_TRY(scope.alloc(&d_nrm, n));
  gather_kernel<<<grid_blocks(ctx, n), kThreads, 0, ctx->stream>>>(c->d_raw, c->d_raw_nrm, d_perm, n, d_pts, d_nrm);
  ctx->launches += 1;
  CB_CUDA(cudaGetLastError());
  // 6. coarse occupancy: the list of non-empty 8x8x8-cell blocks for the far-query path
  uint4* d_blocks = nullptr;
  {
    const int bx = (gp.nx + kBlockCells - 1) / kBlockCells, by = (gp.ny + kBlockCells - 1) / kBlockCells,
              bz = (gp.nz + kBlockCells - 1) / kBlockCells;
    const size_t nb = (size_t)bx * by * bz;
    uint32_t* d_cnt = nullptr;
    CB_TRY(scope.alloc(&d_cnt, 2 * nb + 2));
    uint32_t* d_flag = d_cnt + nb;  // nb + 2 entries
    block_count_kernel<<<grid_blocks(ctx, (nb + 1) * 32), kThreads, 0, ctx->stream>>>(d_hist, gp.nx, gp.ny, gp.nz, bx, by, bz,
                                                                         d_cnt, d_flag);
    CB_TRY(exclusive_scan_u32(ctx, d_flag, nb + 1, 0u));
    // at most min(nb, n) blocks are non-empty: sized without waiting for the count, which is read back at
    // the final synchronise below
    CB_TRY(scope.alloc(&d_blocks, std::min(nb, n)));
    block_emit_kernel<<<grid_blocks(ctx, nb), kThreads, 0, ctx->stream>>>(d_cnt, d_flag, bx, by, bz, d_blocks);
    ctx->launches += 2;
    CB_CUDA(cudaGetLastError());
    CB_CUDA(cudaMemcpyAsync(&c->nblocks, d_flag + nb, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  }
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  // the index arrays go to the cloud (its scope frees them in cb_cloud_destroy)
  for (void* p : {(void*)d_hist, (void*)d_pts, (void*)d_nrm, (void*)d_blocks}) scope.move_to(c->mem, p);
  c->d_cell_start = d_hist;  // (ncells + 1) entries
  c->d_pts = d_pts;
  c->d_nrm = d_nrm;
  c->d_blocks = d_blocks;
  c->indexed = true;
  return CB_OK;
}

GridView grid_view(const cb_cloud* c) {
  GridView g;
  g.pts = c->d_pts;
  g.nrm = c->d_nrm;
  g.cell_start = c->d_cell_start;
  g.ox = c->ox;
  g.oy = c->oy;
  g.oz = c->oz;
  g.inv_h = c->inv_h;
  g.h_safe = (1.0f / c->inv_h) * (1.0f - 0.0009765625f);
  // The one scale factor of every pruning bound (gap^2 * hs2, gap in cells). A point beyond a gap g lies at
  // least (g + 2^-11) h away, so a bound only has to stay at or below its fp32 d2:
  //  * h_safe^2 above FLT_MAX would be +inf (h > ~1.84e19): inf bounds prune rows holding finite d2, and 0 * inf
  //    is NaN. FLT_MAX < h_safe^2 keeps every bound below the unclamped one, and a bound that still overflows
  //    to inf only covers points whose fp32 d2 is inf as well;
  //  * h_safe^2 below 2^-100 (h < ~8.9e-16): the d2 of a point beyond a face may then be subnormal, where fp32
  //    loses the relative precision the margins rely on. Such grids prune nothing (the searches stay exact and
  //    scan everything they reach).
  const float hs = g.h_safe * g.h_safe;
  g.hs2 = hs < 0x1p-100f ? 0.f : fminf(hs, FLT_MAX);
  g.nx = c->nx;
  g.ny = c->ny;
  g.nz = c->nz;
  g.n = (uint32_t)c->n;
  g.blocks = c->d_blocks;
  g.nblocks = c->nblocks;
  return g;
}

}  // namespace cb
