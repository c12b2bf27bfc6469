// Covariance, PCA projection and reconstruction over D-dimensional rows (product code, sm_90a).
//
// Covariance<float, D>::operator() (core/covariance.hpp:30-80) for D != 3 (D = 3 runs the moments kernel of
// stats_kernels.cu on the same bytes). Arithmetic contract (DESIGN §4.18):
//   pivot c = fp32 rounding of the fp64 mean of the first min(n, 4096) rows (a non-finite component is replaced by 0);
//   one pass accumulates S1 = sum (p - c) and S2 = sum (p - c)(p - c)^T in fp64, p - c formed in fp64;
//   mean = c + S1 / n, cov = (S2 - S1 S1^T / n) / (n - 1) in fp64 on the host, rounded to fp32 once.
// S2 is a symmetric rank-n update. The grid is (upper-triangle pairs of T x T output tiles) x (row slabs), slab-major,
// so the tile pairs of one slab run together and read its rows from HBM once. A block stages chunks of its rows for
// the two column tiles as fp64 in shared memory and multiplies them on the FP64 tensor cores (DMMA, mma.sync m8n8k4):
// the order inside an MMA is fixed, so the result does not depend on the run. Every block writes a T x T (+ T for S1)
// partial; a second kernel folds the slabs in ascending order. No atomics.
//
// PrincipalComponentAnalysis::project / reconstruct (core/principal_component_analysis.hpp:46-68): fp32, one rounding
// per operation, no FMA, in the pinned orders
//   project:     acc = 0; for d = 0 .. D-1: acc = acc + E[d][j] * (p_d - mean_d)
//   reconstruct: acc = 0; for j = 0 .. k-1: acc = acc + E[r][j] * q_j;  out_r = acc + mean_r
// tiled like the k-means assignment: 128 rows x 128 outputs per block, an 8 x 8 register tile per thread, the rows and
// the basis staged in shared memory in chunks of 16 input dimensions.
#include "cb_internal.hpp"
#include "launch.cuh"
#include <algorithm>
#include <cmath>
#include <limits>

using namespace cb;

namespace {

constexpr int kCovThreads = 256;    // 8 warps
constexpr int kChunkElems = 2048;   // staged elements per operand and chunk: kRows(T) x T
constexpr int kPivotRows = 4096;    // rows the pivot is the mean of (capi_stats.cu mean_cov_double)

template <int T>
struct CovTile {
  static constexpr int kRows = kChunkElems / T;            // rows per staged chunk (a multiple of 4: MMA k-steps)
  static constexpr int kStride = T == 8 ? 8 : T + 8;       // doubles per staged row: = 8 (mod 16), conflict-free LDS
  static constexpr int kM = T / 8;                         // MMA tiles per tile edge
  static constexpr int kTilesPerWarp = kM * kM >= 8 ? kM * kM / 8 : 1;
  static constexpr int kWarpsK = kM * kM >= 8 ? 1 : 8 / (kM * kM);  // warps splitting the rows of a chunk
  static constexpr int kPerThread = kChunkElems / kCovThreads;   // staged elements per thread and operand
  static constexpr int kPartial = T * T + T;                     // doubles per block partial: S2 tile, then S1
};

// one fp64 8x8x4 MMA: d = a * b + d (A row-major 8x4, B column-major 4x8)
__device__ __forceinline__ void dmma(double (&d)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n"
               : "+d"(d[0]), "+d"(d[1])
               : "d"(a), "d"(b));
}

// (I, J), I <= J, of upper-triangle tile pair p (row-major over I)
__device__ __forceinline__ void tile_pair(int p, int ntiles, int* I, int* J) {
  int i = 0;
  while (p >= ntiles - i) {
    p -= ntiles - i;
    i++;
  }
  *I = i;
  *J = i + p;
}

// Pivot: one block of 32 x 32 threads per 32 dimensions; thread (x, y) sums rows y, y + 32, ... of dimension x in
// fp64, then the 32 row phases are added in ascending order.
__global__ void __launch_bounds__(1024) cov_pivot_kernel(const float* __restrict__ raw, size_t n, int D,
                                                         float* __restrict__ pivot) {
  __shared__ double part[32][33];
  const int d = blockIdx.x * 32 + threadIdx.x;
  const size_t head = n < (size_t)kPivotRows ? n : (size_t)kPivotRows;
  double s = 0.0;
  if (d < D)
    for (size_t r = threadIdx.y; r < head; r += 32) s += (double)raw[r * (size_t)D + d];
  part[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && d < D) {
    double t = 0.0;
    for (int y = 0; y < 32; y++) t += part[y][threadIdx.x];
    const float c = (float)(t / (double)head);
    pivot[d] = isfinite(c) ? c : 0.f;
  }
}

template <int T>
__global__ void __launch_bounds__(kCovThreads) cov_accumulate_kernel(const float* __restrict__ raw, size_t n, int D,
                                                                     const float* __restrict__ pivot, int ntiles,
                                                                     int npairs, size_t slab_rows,
                                                                     double* __restrict__ partials) {
  using P = CovTile<T>;
  extern __shared__ __align__(16) double smem_d[];
  double* sA = smem_d;                            // [kRows][kStride]
  double* sB = smem_d + P::kRows * P::kStride;    // the same for tile J (unused on diagonal pairs)
  const int pair = blockIdx.x % npairs;
  const size_t slab = blockIdx.x / npairs;
  int I, J;
  tile_pair(pair, ntiles, &I, &J);
  const bool diag = I == J;
  const double* sBr = diag ? sA : sB;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const size_t r_lo = slab * slab_rows;
  const size_t r_hi = min(n, r_lo + slab_rows);

  // staging: element e = tid + kCovThreads * i of a chunk is (row e / T, column e % T); kCovThreads % T == 0, so
  // every element of a thread is in the same column
  const int col = tid % T, row0 = tid / T;
  constexpr int kRowStep = kCovThreads / T;
  const int ca = I * T + col, cbj = J * T + col;
  const bool ina = ca < D, inb = cbj < D;
  const double pa = ina ? (double)pivot[ca] : 0.0, pb = inb ? (double)pivot[cbj] : 0.0;
  float ra[P::kPerThread], rb[P::kPerThread];
  auto fetch = [&](size_t c0) {
#pragma unroll
    for (int i = 0; i < P::kPerThread; i++) {
      const size_t r = c0 + row0 + (size_t)i * kRowStep;
      const bool rin = r < r_hi;
      ra[i] = (rin && ina) ? __ldg(raw + r * (size_t)D + ca) : 0.f;
      if (!diag) rb[i] = (rin && inb) ? __ldg(raw + r * (size_t)D + cbj) : 0.f;
    }
  };
  double s1 = 0.0;  // this thread's part of S1 for column ca (diagonal pairs)

  double acc[P::kTilesPerWarp][2];
#pragma unroll
  for (int t = 0; t < P::kTilesPerWarp; t++) acc[t][0] = acc[t][1] = 0.0;
  const int kgroup = warp % P::kWarpsK, tgroup = warp / P::kWarpsK;

  if (r_lo < r_hi) fetch(r_lo);
  for (size_t c0 = r_lo; c0 < r_hi; c0 += P::kRows) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < P::kPerThread; i++) {
      const size_t r = c0 + row0 + (size_t)i * kRowStep;
      const bool rin = r < r_hi;
      // rows past the slab and columns past D are exact zeros: they add nothing to any entry
      const double va = (rin && ina) ? (double)ra[i] - pa : 0.0;
      sA[(row0 + i * kRowStep) * P::kStride + col] = va;
      if (diag) {
        s1 += va;
      } else {
        sB[(row0 + i * kRowStep) * P::kStride + col] = (rin && inb) ? (double)rb[i] - pb : 0.0;
      }
    }
    __syncthreads();
    if (c0 + P::kRows < r_hi) fetch(c0 + P::kRows);
    for (int ks = kgroup; ks < P::kRows / 4; ks += P::kWarpsK) {
      const int kr = ks * 4 + (lane & 3);
#pragma unroll
      for (int t = 0; t < P::kTilesPerWarp; t++) {
        const int tile = tgroup * P::kTilesPerWarp + t;
        const int tm = tile / P::kM, tn = tile % P::kM;
        const double a = sA[kr * P::kStride + tm * 8 + (lane >> 2)];
        const double b = sBr[kr * P::kStride + tn * 8 + (lane >> 2)];
        dmma(acc[t], a, b);
      }
    }
  }

  // the warps' fragments (and the warp row groups of narrow tiles) to shared memory, then added in ascending group
  // order into this block's partial
  __syncthreads();
  double* red = smem_d;  // [kWarpsK][T][T], fits in the staging buffers
#pragma unroll
  for (int t = 0; t < P::kTilesPerWarp; t++) {
    const int tile = tgroup * P::kTilesPerWarp + t;
    const int tm = tile / P::kM, tn = tile % P::kM;
    const int r = tm * 8 + (lane >> 2), c = tn * 8 + 2 * (lane & 3);
    red[(kgroup * T + r) * T + c] = acc[t][0];
    red[(kgroup * T + r) * T + c + 1] = acc[t][1];
  }
  double* s1_part = smem_d + P::kWarpsK * T * T;  // [kRowStep][T]
  s1_part[row0 * T + col] = s1;
  __syncthreads();
  double* out = partials + (slab * npairs + pair) * (size_t)P::kPartial;
  for (int e = tid; e < T * T; e += kCovThreads) {
    double v = red[e];
    for (int g = 1; g < P::kWarpsK; g++) v += red[g * T * T + e];
    out[e] = v;
  }
  if (tid < T) {
    double v = s1_part[tid];
    for (int g = 1; g < kRowStep; g++) v += s1_part[g * T + tid];
    out[T * T + tid] = v;
  }
}

// folded[e] = sum over slabs s = 0 .. nslabs-1, ascending, of partials[s][e]
__global__ void cov_fold_kernel(const double* __restrict__ partials, size_t per_slab, int nslabs,
                                double* __restrict__ folded) {
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < per_slab; e += (size_t)gridDim.x * blockDim.x) {
    double v = 0.0;
    for (int s = 0; s < nslabs; s++) v += partials[(size_t)s * per_slab + e];
    folded[e] = v;
  }
}

// rows[i] = src[idx[i]] (D floats each)
__global__ void gather_rows_kernel(const float* __restrict__ src, int D, const uint64_t* __restrict__ idx, size_t m,
                                   float* __restrict__ rows) {
  const size_t total = m * (size_t)D;
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t i = e / (size_t)D, j = e - i * (size_t)D;
    rows[e] = src[idx[i] * (size_t)D + j];
  }
}

// ---- projection / reconstruction --------------------------------------------------------------------------------
constexpr int kPThreads = 256;       // 16 x 16 threads; thread (ty, tx) owns 8 rows x 8 outputs of a tile
constexpr int kPTile = 128;          // rows and outputs per tile
constexpr int kPChunk = 16;          // input dimensions per staged chunk
constexpr int kPStride = kPTile + 4;

struct PStaging {
  float x[kPChunk][kPStride];  // input rows of the tile, [input dim][row] (projection: already centred)
  float w[kPChunk][kPStride];  // basis, [input dim][output]
};

__device__ __forceinline__ int pslot(int t, int u) { return u < 4 ? t * 4 + u : 64 + t * 4 + (u - 4); }

// in: n x din rows; out: n x dout. Weight of (input a, output b) is E[a * sa + b * sb] (E row-major D x D).
// kProject: x_a = in_a - mean_a before the fold; else out_b = fold + mean_b.
template <bool kProject>
__global__ void __launch_bounds__(kPThreads, 2)
    pca_map_kernel(const float* __restrict__ in, size_t n, int din, int dout, const float* __restrict__ E, int sa,
                   int sb, const float* __restrict__ mean, float* __restrict__ out) {
  __shared__ __align__(16) PStaging st;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const size_t nrt = (n + kPTile - 1) / kPTile;
  const int nct = (dout + kPTile - 1) / kPTile;
  for (size_t t = blockIdx.x; t < nrt * (size_t)nct; t += gridDim.x) {
    const size_t base = (t / nct) * kPTile;
    const int c0 = (int)(t % nct) * kPTile;
    const int rows = (int)min((size_t)kPTile, n - base), cn = min(kPTile, dout - c0);
    float acc[8][8];
#pragma unroll
    for (int u = 0; u < 8; u++)
#pragma unroll
      for (int v = 0; v < 8; v++) acc[u][v] = 0.f;
    for (int lo = 0; lo < din; lo += kPChunk) {
      const int dn = min(kPChunk, din - lo);
      __syncthreads();
      for (int e = threadIdx.x; e < kPTile * dn; e += kPThreads) {
        const int r = e / dn, dd = e - r * dn;
        float v = 0.f;
        if (r < rows) {
          v = in[(base + r) * (size_t)din + lo + dd];
          if (kProject) v = __fsub_rn(v, mean[lo + dd]);
        }
        st.x[dd][r] = v;
      }
      for (int e = threadIdx.x; e < kPTile * dn; e += kPThreads) {
        const int dd = e / kPTile, b = e - dd * kPTile;
        st.w[dd][b] = b < cn ? E[(size_t)(lo + dd) * sa + (size_t)(c0 + b) * sb] : 0.f;
      }
      __syncthreads();
#pragma unroll 2
      for (int dd = 0; dd < dn; dd++) {
        const float4 xa = *reinterpret_cast<const float4*>(&st.x[dd][ty * 4]);
        const float4 xb = *reinterpret_cast<const float4*>(&st.x[dd][64 + ty * 4]);
        const float4 wa = *reinterpret_cast<const float4*>(&st.w[dd][tx * 4]);
        const float4 wb = *reinterpret_cast<const float4*>(&st.w[dd][64 + tx * 4]);
        const float x[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
        const float w[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w};
#pragma unroll
        for (int u = 0; u < 8; u++)
#pragma unroll
          for (int v = 0; v < 8; v++) acc[u][v] = __fadd_rn(acc[u][v], __fmul_rn(w[v], x[u]));
      }
    }
#pragma unroll
    for (int u = 0; u < 8; u++) {
      const int r = pslot(ty, u);
      if (r >= rows) continue;
#pragma unroll
      for (int v = 0; v < 8; v++) {
        const int b = pslot(tx, v);
        if (b >= cn) continue;
        out[(base + r) * (size_t)dout + c0 + b] = kProject ? acc[u][v] : __fadd_rn(acc[u][v], mean[c0 + b]);
      }
    }
  }
}

template <int T>
int cov_launch(cb_context* ctx, const float* raw, size_t n, int D, const float* d_pivot, DeviceScope& scope,
               double* h_folded, int* ntiles_out) {
  using P = CovTile<T>;
  const int ntiles = (D + T - 1) / T;
  const int npairs = ntiles * (ntiles + 1) / 2;
  // enough slabs for about four blocks per SM, no slab shorter than one chunk
  const size_t chunks = std::max<size_t>(1, (n + P::kRows - 1) / P::kRows);
  const size_t want = std::max<size_t>(1, ((size_t)ctx->sm_count * 4 + npairs - 1) / npairs);
  const size_t nslabs0 = std::min(chunks, want);
  const size_t slab_rows = ((chunks + nslabs0 - 1) / nslabs0) * P::kRows;
  const size_t nslabs = std::max<size_t>(1, (n + slab_rows - 1) / slab_rows);
  const size_t per_slab = (size_t)npairs * P::kPartial;
  double *d_part = nullptr, *d_fold = nullptr;
  CB_TRY(scope.alloc(&d_part, nslabs * per_slab));
  CB_TRY(scope.alloc(&d_fold, per_slab));
  const size_t smem = 2 * (size_t)P::kRows * P::kStride * sizeof(double);
  static_assert(P::kWarpsK * T * T + (kCovThreads / T) * T <= 2 * P::kRows * P::kStride, "reduction fits the staging");
  CB_CUDA(cudaFuncSetAttribute(cov_accumulate_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CB_TRY(launch(ctx, cov_accumulate_kernel<T>, dim3((unsigned)(nslabs * npairs)), kCovThreads, smem, raw, n, D,
                d_pivot, ntiles, npairs, slab_rows, d_part));
  CB_TRY(launch(ctx, cov_fold_kernel, grid_for(ctx, per_slab, 256), 256, 0, d_part, per_slab, (int)nslabs, d_fold));
  CB_CUDA(cudaMemcpyAsync(h_folded, d_fold, per_slab * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  *ntiles_out = ntiles;
  return CB_OK;
}

}  // namespace

namespace cb {

static int cov_tile_edge(int D) { return D <= 8 ? 8 : D <= 16 ? 16 : D <= 32 ? 32 : 64; }

int vectors_gather(cb_context* ctx, const float* raw, int D, const uint64_t* d_idx, size_t m, float* rows) {
  return launch(ctx, gather_rows_kernel, grid_for(ctx, m * (size_t)D, 256), 256, 0, raw, D, d_idx, m, rows);
}

int features_mean_cov(cb_context* ctx, const float* raw, size_t n, int D, float* mean, float* cov) {
  DeviceScope scope(ctx);
  float* d_pivot = nullptr;
  CB_TRY(scope.alloc(&d_pivot, (size_t)D));
  CB_TRY(launch(ctx, cov_pivot_kernel, dim3((unsigned)((D + 31) / 32)), dim3(32, 32), 0, raw, n, D, d_pivot));
  const int T = cov_tile_edge(D);
  const int nt = (D + T - 1) / T;
  std::vector<double> folded((size_t)nt * (nt + 1) / 2 * (T * T + T));
  std::vector<float> pivot((size_t)D);
  int ntiles = 0;
  switch (T) {
    case 8: CB_TRY(cov_launch<8>(ctx, raw, n, D, d_pivot, scope, folded.data(), &ntiles)); break;
    case 16: CB_TRY(cov_launch<16>(ctx, raw, n, D, d_pivot, scope, folded.data(), &ntiles)); break;
    case 32: CB_TRY(cov_launch<32>(ctx, raw, n, D, d_pivot, scope, folded.data(), &ntiles)); break;
    default: CB_TRY(cov_launch<64>(ctx, raw, n, D, d_pivot, scope, folded.data(), &ntiles)); break;
  }
  CB_CUDA(cudaMemcpyAsync(pivot.data(), d_pivot, (size_t)D * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  // the folded tile pairs, row-major over I <= J: S2 in the first T x T doubles, S1 after them on diagonal pairs
  std::vector<size_t> pair_base((size_t)ntiles * ntiles);
  for (int I = 0, p = 0; I < ntiles; I++)
    for (int J = I; J < ntiles; J++, p++) pair_base[(size_t)I * ntiles + J] = (size_t)p * (T * T + T);
  const double nn = (double)n;
  std::vector<double> s1((size_t)D);
  for (int j = 0; j < D; j++) {
    const int I = j / T;
    s1[j] = folded[pair_base[(size_t)I * ntiles + I] + (size_t)T * T + (j % T)];
    mean[j] = (float)((double)pivot[j] + s1[j] / nn);
  }
  for (int i = 0; i < D; i++)
    for (int j = i; j < D; j++) {
      const double s2 = folded[pair_base[(size_t)(i / T) * ntiles + j / T] + (size_t)(i % T) * T + (j % T)];
      // a non-finite value in dimension i or j makes S1_i or S1_j non-finite (fp32 inputs cannot overflow the fp64
      // sums): row and column of that dimension are NaN, as the reference's two passes give
      const float v = (std::isfinite(s1[i]) && std::isfinite(s1[j]))
                          ? (float)((s2 - s1[i] * s1[j] / nn) / (nn - 1.0))
                          : std::numeric_limits<float>::quiet_NaN();
      cov[(size_t)i * D + j] = cov[(size_t)j * D + i] = v;
    }
  return CB_OK;
}

int features_map(cb_context* ctx, const float* in, size_t n, int din, int dout, const float* d_E, int sa, int sb,
                 const float* d_mean, bool project, float* out) {
  const size_t tiles = ((n + kPTile - 1) / kPTile) * (size_t)((dout + kPTile - 1) / kPTile);
  const int grid = (int)std::max<size_t>(1, std::min<size_t>(tiles, (size_t)ctx->sm_count * 2));
  if (project)
    return launch(ctx, pca_map_kernel<true>, grid, kPThreads, 0, in, n, din, dout, d_E, sa, sb, d_mean, out);
  return launch(ctx, pca_map_kernel<false>, grid, kPThreads, 0, in, n, din, dout, d_E, sa, sb, d_mean, out);
}

}  // namespace cb
