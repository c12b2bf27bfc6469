// Classical multidimensional scaling over an n x n distance matrix (product code, sm_90a).
//
// computeDistancePreservingSpectralEmbedding (utilities/multidimensional_scaling.hpp:35-83) under the contract of
// DESIGN §4.19. E_ij is the entry of the n x n fp32 matrix Dm, squared once in fp32 when the distances are not squared.
// B is the symmetric matrix whose entries for i >= j are -1/2 (E_ij - r_i - c_j + g) (r row means, c column means, g
// grand mean, all fp64): -1/2 J E J restricted to the lower triangle, the triangle the reference's eigen-solver reads.
// Neither J nor B is formed. The kernels:
//   means:   one read of E gives the fp64 row and column sums (slab partials folded in a fixed order), then g and
//            rg_i = g - r_i;
//   product: Y = B X for an n x 8 or n x 16 fp64 block X. A block owns a strip of 256 rows and a run of 32-column
//            chunks of the lower triangle; it stages each chunk with its rows of X and c (cp.async, and the strip's
//            rows of X once), forms every B entry in registers from E, rg and c, and multiplies on the FP64 tensor
//            cores (mma.sync m8n8k4): the strip side Y_I += B_IJ X_J stays in
//            the accumulators across the run, the chunk side Y_J += B_IJ^T X_I is folded over the 8 warps in ascending
//            order and written per chunk. A fold kernel adds a row's strip partials and then its chunk partials in
//            ascending strip order. No atomics: the same X gives the same bits;
//   gram / combine: G = A^T Z (slab partials, fixed fold) and Z (+)= A C for the n x m basis, row-major.
// The solver on the host is a restarted block Krylov iteration with Rayleigh-Ritz (DESIGN §4.19).
#include "cb_internal.hpp"
#include "launch.cuh"
#include <algorithm>
#include <cmath>
#include <limits>
#include <numeric>
#include <type_traits>
#include <vector>

using namespace cb;

namespace {

constexpr int kThreads = 256;  // 8 warps
constexpr int kStrip = 256;    // rows per product strip (32 per warp)
constexpr int kChunk = 32;     // columns per staged chunk
constexpr int kStride = 36;    // floats per staged row: conflict-free strip-side fragment loads
constexpr int kStages = 2;     // staged chunks per block (3 or 4 measured within 2 %: the product is not latency-bound)
constexpr int kMeansCols = 1024;  // columns per means block (4 per thread)
constexpr int kMeansRows = 64;    // rows per means slab

__device__ __forceinline__ void dmma(double (&d)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n"
               : "+d"(d[0]), "+d"(d[1])
               : "d"(a), "d"(b));
}

__device__ __forceinline__ void cp_async_4(float* dst, const float* src, bool in) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(s), "l"(src), "r"(in ? 4 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_16(float* dst, const float* src, bool in) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(src), "r"(in ? 16 : 0) : "memory");
}
// 16-byte copy of which the first `bytes` come from src and the rest are zero
__device__ __forceinline__ void cp_async_16_part(float* dst, const float* src, unsigned bytes) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory");
}

template <bool kSquare>
__device__ __forceinline__ float entry(float x) {
  return kSquare ? __fmul_rn(x, x) : x;
}

// ---- means ------------------------------------------------------------------------------------------------------
// Block (column chunk, row slab): thread t sums columns chunk * 1024 + t + 256 k (k = 0..3) over the slab's rows into
// colpart[slab][col]; each row's 1024 values are added per thread (k ascending), over the warp (xor butterfly) and over
// the 8 warps (ascending) into rowpart[chunk][row].
template <bool kSquare>
__global__ void __launch_bounds__(kThreads) mds_means_kernel(const float* __restrict__ dm, size_t n,
                                                             double* __restrict__ rowpart, double* __restrict__ colpart) {
  __shared__ double wsum[kThreads / 32][kMeansRows];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const size_t chunk = blockIdx.x, slab = blockIdx.y;
  const size_t r0 = slab * kMeansRows, r1 = min(n, r0 + kMeansRows);
  double cs[4] = {0.0, 0.0, 0.0, 0.0};
  for (size_t r = r0; r < r1; r++) {
    double rs = 0.0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const size_t c = chunk * kMeansCols + t + 256 * k;
      const double v = c < n ? (double)entry<kSquare>(__ldg(dm + r * n + c)) : 0.0;
      cs[k] += v;
      rs += v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, o);
    if (lane == 0) wsum[warp][r - r0] = rs;
  }
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const size_t c = chunk * kMeansCols + t + 256 * k;
    if (c < n) colpart[slab * n + c] = cs[k];
  }
  __syncthreads();
  if ((size_t)t < r1 - r0) {
    double v = wsum[0][t];
    for (int w = 1; w < kThreads / 32; w++) v += wsum[w][t];
    rowpart[chunk * n + r0 + t] = v;
  }
}

// sums[i] = row sum i (chunks ascending), sums[n + j] = column sum j (slabs ascending)
__global__ void mds_means_fold_kernel(const double* __restrict__ rowpart, const double* __restrict__ colpart, size_t n,
                                      int nchunks, int nslabs, double* __restrict__ sums) {
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < 2 * n; e += (size_t)gridDim.x * blockDim.x) {
    double v = 0.0;
    if (e < n)
      for (int k = 0; k < nchunks; k++) v += rowpart[(size_t)k * n + e];
    else
      for (int s = 0; s < nslabs; s++) v += colpart[(size_t)s * n + (e - n)];
    sums[e] = v;
  }
}

// One block of 1024 threads: g = (sum of the row sums) / n^2 (thread strides, then a fixed tree), then
// rg_i = g - r_i and c_j = colsum_j / n. g goes to out_g.
__global__ void __launch_bounds__(1024) mds_means_finish_kernel(const double* __restrict__ sums, size_t n,
                                                                double* __restrict__ rg, double* __restrict__ cm,
                                                                double* __restrict__ out_g) {
  __shared__ double red[1024];
  const int t = threadIdx.x;
  double s = 0.0;
  for (size_t i = t; i < n; i += 1024) s += sums[i];
  red[t] = s;
  __syncthreads();
  for (int w = 512; w > 0; w >>= 1) {
    if (t < w) red[t] += red[t + w];
    __syncthreads();
  }
  const double nn = (double)n;
  const double g = red[0] / nn / nn;
  for (size_t i = t; i < n; i += 1024) {
    rg[i] = g - sums[i] / nn;
    cm[i] = sums[n + i] / nn;
  }
  if (t == 0) *out_g = g;
}

// ---- Y = B X ----------------------------------------------------------------------------------------------------
struct ProductWork {
  const int* blk_strip;   // [blocks] strip of each block
  const int* blk_q0;      // [blocks] first chunk of each block's run
  const int* blk_q1;      // [blocks] one past its last chunk
  const int* strip_blk0;  // [nstrips + 1] first block of each strip
  const size_t* strip_chunk0;  // [nstrips] first chunk-partial slot of each strip
  int nstrips;
};

// Staged chunk: kStrip rows x kChunk columns of E, [row][col] with kStride floats per row.
template <int NB, bool kSquare>
__global__ void __launch_bounds__(kThreads, 1)
    mds_product_kernel(const float* __restrict__ dm, size_t n, const double* __restrict__ rg,
                       const double* __restrict__ cm, const double* __restrict__ X, int ldx, ProductWork wk,
                       double* __restrict__ prow, double* __restrict__ pcol) {
  constexpr int BW = NB * 8;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int XS = BW + 4;  // doubles per staged X row: conflict-free fragment loads at both widths
  float* st = reinterpret_cast<float*>(smem_raw);                           // [kStages][kStrip][kStride]
  double* red = reinterpret_cast<double*>(st + kStages * kStrip * kStride);  // [8 warps][kChunk][BW]
  double* xis = red + 8 * kChunk * BW;                                       // [kStrip][XS]: X_I, the strip's rows
  double* xjs = xis + kStrip * XS;                                           // [kStages][kChunk][XS]: X_J
  double* cjs_s = xjs + kStages * kChunk * XS;                               // [kStages][kChunk]: c_J
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int I = wk.blk_strip[blockIdx.x];
  const int q0 = wk.blk_q0[blockIdx.x], q1 = wk.blk_q1[blockIdx.x];
  const size_t row0 = (size_t)I * kStrip;
  const int la = lane >> 2, lb = lane & 3;

  // staging: with n % 4 == 0 every row of a chunk is 16-byte aligned and thread tid copies the 4 columns
  // 4 (tid % 8) .. + 3 of rows tid / 8 + 32 k; otherwise column tid % 32 of rows tid / 32 + 8 k, one float at a time
  const bool vec4 = (n & 3) == 0;
  auto issue = [&](int q, int buf) {
    float* dst = st + buf * kStrip * kStride;
    {  // the chunk's X rows and column means, 16 bytes a copy (zero past n)
      const size_t col0 = (size_t)q * kChunk;
      for (int e = tid; e < kChunk * BW / 2; e += kThreads) {
        const int r = e / (BW / 2), h = e % (BW / 2);
        const bool in = col0 + r < n;
        cp_async_16(reinterpret_cast<float*>(xjs + (buf * kChunk + r) * XS + 2 * h),
                    reinterpret_cast<const float*>(in ? X + (col0 + r) * ldx + 2 * h : X), in);
      }
      if (tid < kChunk / 2) {
        const size_t j = col0 + 2 * tid;
        const unsigned bytes = j + 1 < n ? 16u : j < n ? 8u : 0u;
        cp_async_16_part(reinterpret_cast<float*>(cjs_s + buf * kChunk + 2 * tid),
                         reinterpret_cast<const float*>(bytes ? cm + j : cm), bytes);
      }
    }
    if (vec4) {
      const size_t c = (size_t)q * kChunk + 4 * (tid & 7);
#pragma unroll
      for (int k = 0; k < kStrip / 32; k++) {
        const int rr = (tid >> 3) + 32 * k;
        const size_t r = row0 + rr;
        const bool in = r < n && c < n;
        cp_async_16(dst + rr * kStride + 4 * (tid & 7), in ? dm + r * n + c : dm, in);
      }
      return;
    }
    const size_t c = (size_t)q * kChunk + (tid & 31);
#pragma unroll 8
    for (int k = 0; k < kStrip / 8; k++) {
      const int rr = (tid >> 5) + 8 * k;
      const size_t r = row0 + rr;
      const bool in = r < n && c < n;
      cp_async_4(dst + rr * kStride + (tid & 31), in ? dm + r * n + c : dm, in);
    }
  };

  // per-block constants: the rows of this warp in strip-side (a) and chunk-side (b) fragment positions
  const int wr = warp * 32;
  double rg_a[4], rg_b[8];
  bool in_a[4], in_b[8];
#pragma unroll
  for (int tr = 0; tr < 4; tr++) {
    const size_t i = row0 + wr + 8 * tr + la;
    in_a[tr] = i < n;
    rg_a[tr] = in_a[tr] ? rg[i] : 0.0;
  }
#pragma unroll
  for (int ks = 0; ks < 8; ks++) {
    const size_t i = row0 + wr + 4 * ks + lb;
    in_b[ks] = i < n;
    rg_b[ks] = in_b[ks] ? rg[i] : 0.0;
  }
  double acc_i[4][NB][2];
#pragma unroll
  for (int tr = 0; tr < 4; tr++)
#pragma unroll
    for (int g = 0; g < NB; g++) acc_i[tr][g][0] = acc_i[tr][g][1] = 0.0;

  for (int e = tid; e < kStrip * BW / 2; e += kThreads) {  // X_I, in the first copy group
    const int r = e / (BW / 2), h = e % (BW / 2);
    const bool in = row0 + r < n;
    cp_async_16(reinterpret_cast<float*>(xis + r * XS + 2 * h),
                reinterpret_cast<const float*>(in ? X + (row0 + r) * ldx + 2 * h : X), in);
  }
  for (int t = 0; t < kStages - 1; t++) {
    if (q0 + t < q1) issue(q0 + t, t);
    cp_async_commit();
  }
  for (int q = q0; q < q1; q++) {
    const int buf = (q - q0) % kStages;
    cp_async_wait<kStages - 2>();
    __syncthreads();
    // into the buffer of chunk q - 1, free since every thread passed the barrier above
    if (q + kStages - 1 < q1) issue(q + kStages - 1, (q - q0 + kStages - 1) % kStages);
    cp_async_commit();
    const float* s = st + buf * kStrip * kStride;
    const double* xj_s = xjs + buf * kChunk * XS;
    const double* cj_s = cjs_s + buf * kChunk;
    const size_t col0 = (size_t)q * kChunk;
    double acc_j[4][NB][2];
    // kMasked: the chunk crosses the diagonal or the matrix edge, so entries are tested; a chunk wholly below the
    // strip's first row and inside the matrix needs no test
    auto body = [&](auto masked) {
      constexpr bool kMasked = decltype(masked)::value;
      // strip side: A = B[i][j], i = row of this warp's tile tr, j = col0 + 4 ks + lb; B operand X_J
#pragma unroll 2
      for (int ks = 0; ks < 8; ks++) {
        const size_t j = col0 + 4 * ks + lb;
        const bool jin = !kMasked || j < n;
        const double cj = cj_s[4 * ks + lb];  // zero past n
        double xj[NB];
#pragma unroll
        for (int g = 0; g < NB; g++) xj[g] = xj_s[(4 * ks + lb) * XS + g * 8 + la];
#pragma unroll
        for (int tr = 0; tr < 4; tr++) {
          const int rr = wr + 8 * tr + la;
          const double e = ((double)entry<kSquare>(s[rr * kStride + 4 * ks + lb]) - cj) + rg_a[tr];
          const double a = (!kMasked || (jin && in_a[tr] && row0 + rr >= j)) ? e : 0.0;
#pragma unroll
          for (int g = 0; g < NB; g++) dmma(acc_i[tr][g], a, xj[g]);
        }
      }
      // chunk side: A = B^T[j][i] = B[i][j], j = col0 + 8 tc + la, i = row0 + wr + 4 ks + lb; B operand X_I
      double cjs[4];
#pragma unroll
      for (int tc = 0; tc < 4; tc++) {
        cjs[tc] = cj_s[8 * tc + la];
#pragma unroll
        for (int g = 0; g < NB; g++) acc_j[tc][g][0] = acc_j[tc][g][1] = 0.0;
      }
#pragma unroll
      for (int ks = 0; ks < 8; ks++) {
        const int rr = wr + 4 * ks + lb;
        double xi[NB];  // X_I rows of this warp (zero past n)
#pragma unroll
        for (int g = 0; g < NB; g++) xi[g] = xis[rr * XS + g * 8 + la];
#pragma unroll
        for (int tc = 0; tc < 4; tc++) {
          const size_t j = col0 + 8 * tc + la;
          const double e = ((double)entry<kSquare>(s[rr * kStride + 8 * tc + la]) - cjs[tc]) + rg_b[ks];
          const double a = (!kMasked || (j < n && in_b[ks] && row0 + rr > j)) ? e : 0.0;
#pragma unroll
          for (int g = 0; g < NB; g++) dmma(acc_j[tc][g], a, xi[g]);
        }
      }
    };
    if (col0 + kChunk <= row0 && row0 + kStrip <= n)
      body(std::false_type{});
    else
      body(std::true_type{});
#pragma unroll
    for (int tc = 0; tc < 4; tc++)
#pragma unroll
      for (int g = 0; g < NB; g++) {
        const int r = 8 * tc + la, c = g * 8 + 2 * lb;
        red[(warp * kChunk + r) * BW + c] = acc_j[tc][g][0];
        red[(warp * kChunk + r) * BW + c + 1] = acc_j[tc][g][1];
      }
    __syncthreads();
    double* out = pcol + (wk.strip_chunk0[I] + (size_t)q) * (kChunk * BW);
    for (int e = tid; e < kChunk * BW; e += kThreads) {
      double v = red[e];
#pragma unroll
      for (int w = 1; w < kThreads / 32; w++) v += red[w * kChunk * BW + e];
      out[e] = v;
    }
  }
  double* out = prow + (size_t)blockIdx.x * (kStrip * BW);
#pragma unroll
  for (int tr = 0; tr < 4; tr++)
#pragma unroll
    for (int g = 0; g < NB; g++) {
      const int r = wr + 8 * tr + la, c = g * 8 + 2 * lb;
      out[r * BW + c] = acc_i[tr][g][0];
      out[r * BW + c + 1] = acc_i[tr][g][1];
    }
}

// Y[r][c] = -1/2 (strip partials of r's strip, blocks ascending; then chunk partials of r's chunk, strips ascending)
template <int NB>
__global__ void mds_product_fold_kernel(const double* __restrict__ prow, const double* __restrict__ pcol, size_t n,
                                        ProductWork wk, double* __restrict__ Y, int ldy) {
  constexpr int BW = NB * 8;
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < n * BW; e += (size_t)gridDim.x * blockDim.x) {
    const size_t r = e / BW;
    const int c = (int)(e % BW);
    const int I = (int)(r / kStrip);
    const size_t q = r / kChunk;
    double v = 0.0;
    for (int b = wk.strip_blk0[I]; b < wk.strip_blk0[I + 1]; b++)
      v += prow[(size_t)b * (kStrip * BW) + (r - (size_t)I * kStrip) * BW + c];
    for (int J = I; J < wk.nstrips; J++)
      v += pcol[(wk.strip_chunk0[J] + q) * (kChunk * BW) + (r % kChunk) * BW + c];
    Y[r * ldy + c] = -0.5 * v;
  }
}

// ---- basis algebra ----------------------------------------------------------------------------------------------
// part[slab][p * qz + q] = sum over the slab's rows r of A[r][p] * Z[r][q]
__global__ void mds_gram_kernel(const double* __restrict__ A, int lda, int pa, const double* __restrict__ Z, int ldz,
                                int qz, size_t n, size_t slab_rows, double* __restrict__ part) {
  const size_t outs = (size_t)pa * qz;
  const size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (e >= outs) return;
  const int p = (int)(e / qz), q = (int)(e % qz);
  const size_t r0 = blockIdx.y * slab_rows, r1 = min(n, r0 + slab_rows);
  double v = 0.0;
  for (size_t r = r0; r < r1; r++) v += A[r * lda + p] * Z[r * ldz + q];
  part[blockIdx.y * outs + e] = v;
}

__global__ void mds_slab_fold_kernel(const double* __restrict__ part, size_t per_slab, int nslabs,
                                     double* __restrict__ out) {
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < per_slab; e += (size_t)gridDim.x * blockDim.x) {
    double v = 0.0;
    for (int s = 0; s < nslabs; s++) v += part[(size_t)s * per_slab + e];
    out[e] = v;
  }
}

// out[r][q] = (accumulate ? out[r][q] : 0) + sum_k A[r][k] * C[k][q]  (C row-major pa x qc; out and A do not overlap)
__global__ void mds_combine_kernel(const double* __restrict__ A, int lda, int pa, const double* __restrict__ C, int qc,
                                   size_t n, bool accumulate, double* out, int ldo) {
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < n * qc; e += (size_t)gridDim.x * blockDim.x) {
    const size_t r = e / qc;
    const int q = (int)(e % qc);
    double v = 0.0;
    for (int k = 0; k < pa; k++) v += A[r * lda + k] * C[(size_t)k * qc + q];
    out[r * ldo + q] = accumulate ? out[r * ldo + q] + v : v;
  }
}

// ---- host solver ------------------------------------------------------------------------------------------------
uint64_t splitmix64(uint64_t& s) {
  uint64_t z = (s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
double uniform_pm1(uint64_t& s) { return (double)(splitmix64(s) >> 11) * 0x1.0p-52 - 1.0; }

struct Solver {
  cb_context* ctx;
  DeviceScope& scope;
  const float* dm;
  size_t n;
  bool square;
  int bp = 8;     // padded block width (a multiple of 8)
  int b = 8;      // real block width
  int s = 1;      // blocks in the basis
  int M = 8;      // buffer columns: s * bp
  double *V = nullptr, *W = nullptr, *Z = nullptr, *Z2 = nullptr;  // n x M, n x M, n x bp, n x bp
  double *rg = nullptr, *cm = nullptr;
  double *part = nullptr, *small = nullptr, *prow = nullptr, *pcol = nullptr;
  size_t part_cap = 0, small_cap = 0;
  ProductWork wk{};
  int pblocks = 0;
  uint64_t rng = 0x243F6A8885A308D3ull;

  Solver(cb_context* c, DeviceScope& sc, const float* d, size_t n_, bool sq) : ctx(c), scope(sc), dm(d), n(n_), square(sq) {}

  int setup_product() {
    const int nstrips = (int)((n + kStrip - 1) / kStrip);
    const int nchunks = (int)((n + kChunk - 1) / kChunk);
    std::vector<int> nch((size_t)nstrips);
    size_t total = 0;
    for (int I = 0; I < nstrips; I++) {
      nch[I] = std::min(nchunks, (I + 1) * (kStrip / kChunk));
      total += (size_t)nch[I];
    }
    // runs long enough that the strip-side partial is small beside the chunks, about four blocks per SM
    const int run = (int)std::max<size_t>(4, (total + 4 * (size_t)ctx->sm_count - 1) / (4 * (size_t)ctx->sm_count));
    std::vector<int> bs, b0, b1, sb0((size_t)nstrips + 1);
    std::vector<size_t> sc0((size_t)nstrips);
    size_t slot = 0;
    for (int I = 0; I < nstrips; I++) {
      sb0[I] = (int)bs.size();
      sc0[I] = slot;
      for (int q = 0; q < nch[I]; q += run) {
        bs.push_back(I);
        b0.push_back(q);
        b1.push_back(std::min(nch[I], q + run));
      }
      slot += (size_t)nch[I];
    }
    sb0[nstrips] = (int)bs.size();
    pblocks = (int)bs.size();
    int *d_bs, *d_b0, *d_b1, *d_sb0;
    size_t* d_sc0;
    CB_TRY(scope.alloc(&d_bs, bs.size()));
    CB_TRY(scope.alloc(&d_b0, bs.size()));
    CB_TRY(scope.alloc(&d_b1, bs.size()));
    CB_TRY(scope.alloc(&d_sb0, sb0.size()));
    CB_TRY(scope.alloc(&d_sc0, sc0.size()));
    CB_CUDA(cudaMemcpyAsync(d_bs, bs.data(), bs.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    CB_CUDA(cudaMemcpyAsync(d_b0, b0.data(), b0.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    CB_CUDA(cudaMemcpyAsync(d_b1, b1.data(), b1.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    CB_CUDA(cudaMemcpyAsync(d_sb0, sb0.data(), sb0.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    CB_CUDA(cudaMemcpyAsync(d_sc0, sc0.data(), sc0.size() * sizeof(size_t), cudaMemcpyHostToDevice, ctx->stream));
    wk = ProductWork{d_bs, d_b0, d_b1, d_sb0, d_sc0, nstrips};
    CB_TRY(scope.alloc(&prow, (size_t)pblocks * kStrip * 16));
    CB_TRY(scope.alloc(&pcol, slot * kChunk * 16));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));  // the host tables above are freed on return
    return CB_OK;
  }

  template <int NB, bool kSq>
  int product_slice(const double* X, int ldx, double* Y, int ldy) {
    constexpr int BW = NB * 8, XS = BW + 4;
    const size_t smem = (size_t)kStages * kStrip * kStride * sizeof(float) +
                        ((size_t)8 * kChunk * BW + (size_t)kStrip * XS + (size_t)kStages * kChunk * (XS + 1)) *
                            sizeof(double);
    CB_CUDA(cudaFuncSetAttribute(mds_product_kernel<NB, kSq>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CB_TRY(launch(ctx, mds_product_kernel<NB, kSq>, dim3((unsigned)pblocks), kThreads, smem, dm, n, rg, cm, X, ldx, wk,
                  prow, pcol));
    return launch(ctx, mds_product_fold_kernel<NB>, grid_for(ctx, n * NB * 8, 256), 256, 0, prow, pcol, n, wk, Y, ldy);
  }

  // W[:, c0 : c0 + bp] = B V[:, c0 : c0 + bp], in slices of 16 (and a last one of 8) columns
  int product(int c0) {
    for (int c = 0; c < bp; c += 16) {
      const bool wide = bp - c >= 16;
      if (square) {
        if (wide) CB_TRY((product_slice<2, true>(V + c0 + c, M, W + c0 + c, M)));
        else CB_TRY((product_slice<1, true>(V + c0 + c, M, W + c0 + c, M)));
      } else {
        if (wide) CB_TRY((product_slice<2, false>(V + c0 + c, M, W + c0 + c, M)));
        else CB_TRY((product_slice<1, false>(V + c0 + c, M, W + c0 + c, M)));
      }
    }
    return CB_OK;
  }

  int ensure(double** p, size_t* cap, size_t count) {
    if (count <= *cap) return CB_OK;
    if (*p) CB_TRY(scope.free(*p));
    CB_TRY(scope.alloc(p, count));
    *cap = count;
    return CB_OK;
  }

  // G (pa x qz, host) = A^T Z
  int gram(const double* A, int lda, int pa, const double* Zp, int ldz, int qz, std::vector<double>& G) {
    const size_t outs = (size_t)pa * qz;
    const unsigned gx = (unsigned)((outs + 255) / 256);
    const size_t want = std::max<size_t>(1, (size_t)ctx->sm_count * 8 / gx);
    const size_t slab_rows = std::max<size_t>(64, (n + want - 1) / want);
    const int nslabs = (int)((n + slab_rows - 1) / slab_rows);
    CB_TRY(ensure(&part, &part_cap, (size_t)nslabs * outs + outs));
    CB_TRY(launch(ctx, mds_gram_kernel, dim3(gx, (unsigned)nslabs), 256, 0, A, lda, pa, Zp, ldz, qz, n, slab_rows,
                  part));
    double* fold = part + (size_t)nslabs * outs;
    CB_TRY(launch(ctx, mds_slab_fold_kernel, grid_for(ctx, outs, 256), 256, 0, part, outs, nslabs, fold));
    G.resize(outs);
    CB_CUDA(cudaMemcpyAsync(G.data(), fold, outs * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    return CB_OK;
  }

  // out (+)= A C, C host pa x qc
  int combine(const double* A, int lda, int pa, const std::vector<double>& C, int qc, bool accumulate, double* out,
              int ldo) {
    CB_TRY(ensure(&small, &small_cap, C.size()));
    CB_CUDA(cudaMemcpyAsync(small, C.data(), C.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    CB_TRY(launch(ctx, mds_combine_kernel, grid_for(ctx, n * qc, 256), 256, 0, A, lda, pa, small, qc, n, accumulate,
                  out, ldo));
    return CB_OK;
  }

  int copy_cols(double* dst, int ldd, const double* src, int lds, int cols) {
    CB_CUDA(cudaMemcpy2DAsync(dst, (size_t)ldd * sizeof(double), src, (size_t)lds * sizeof(double),
                              (size_t)cols * sizeof(double), n, cudaMemcpyDeviceToDevice, ctx->stream));
    return CB_OK;
  }

  // random columns (fixed seed sequence) into the listed columns of V block k: one upload of an n x bp block into Z2,
  // then a device copy per column
  int randomize(int k, const std::vector<int>& cols) {
    std::vector<double> h(n * (size_t)bp, 0.0);
    for (int c : cols)
      for (size_t i = 0; i < n; i++) h[i * bp + c] = uniform_pm1(rng);
    CB_CUDA(cudaMemcpyAsync(Z2, h.data(), h.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    for (int c : cols) CB_TRY(copy_cols(V + (size_t)k * bp + c, M, Z2 + c, bp, 1));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));  // h is freed on return
    return CB_OK;
  }

  // upper-triangular R with G = R^T R over the first b rows / columns of the bp x bp G, and R^-1 (bp x bp, zero
  // outside b x b). Column j is deficient when its pivot keeps less than 1e-12 of the norm ref[j] it had.
  static std::vector<int> cholesky_inverse(const std::vector<double>& G, int bp, int b, const std::vector<double>& ref,
                                           std::vector<double>& Rinv) {
    std::vector<double> R((size_t)b * b, 0.0);
    std::vector<int> bad;
    for (int j = 0; j < b; j++) {
      double d = G[(size_t)j * bp + j];
      for (int k = 0; k < j; k++) d -= R[(size_t)k * b + j] * R[(size_t)k * b + j];
      if (!(d > 1e-24 * ref[j]) || !(d > 0.0)) {
        bad.push_back(j);
        R[(size_t)j * b + j] = 1.0;
        continue;
      }
      const double rjj = std::sqrt(d);
      R[(size_t)j * b + j] = rjj;
      for (int l = j + 1; l < b; l++) {
        double v = G[(size_t)j * bp + l];
        for (int k = 0; k < j; k++) v -= R[(size_t)k * b + j] * R[(size_t)k * b + l];
        R[(size_t)j * b + l] = v / rjj;
      }
    }
    Rinv.assign((size_t)bp * bp, 0.0);
    for (int j = b - 1; j >= 0; j--) {  // columns of R^-1 by back substitution
      Rinv[(size_t)j * bp + j] = 1.0 / R[(size_t)j * b + j];
      for (int i = j - 1; i >= 0; i--) {
        double v = 0.0;
        for (int k = i + 1; k <= j; k++) v += R[(size_t)i * b + k] * Rinv[(size_t)k * bp + j];
        Rinv[(size_t)i * bp + j] = -v / R[(size_t)i * b + i];
      }
    }
    return bad;
  }

  // V block k <- an orthonormal basis of its columns' part orthogonal to blocks 0 .. k-1 (two projections, then
  // Cholesky QR twice); deficient columns are replaced by random ones and the block is done again. The partner block
  // of W, when given, gets the same column operations (it holds B times the block).
  int orthonormalize(int k, bool with_w) {
    double* Vk = V + (size_t)k * bp;
    double* Wk = W + (size_t)k * bp;
    const int p = k * bp;
    std::vector<double> G, C, Rinv;
    for (int attempt = 0; attempt < 8; attempt++) {
      std::vector<double> ref((size_t)b);
      CB_TRY(gram(Vk, M, bp, Vk, M, bp, G));
      for (int j = 0; j < b; j++) ref[j] = G[(size_t)j * bp + j];
      for (int pass = 0; pass < 2 && p > 0; pass++) {
        CB_TRY(gram(V, M, p, Vk, M, bp, C));
        for (double& x : C) x = -x;
        CB_TRY(combine(V, M, p, C, bp, true, Vk, M));
        if (with_w) CB_TRY(combine(W, M, p, C, bp, true, Wk, M));
      }
      bool ok = true;
      for (int round = 0; round < 2; round++) {
        CB_TRY(gram(Vk, M, bp, Vk, M, bp, G));
        const std::vector<int> bad = cholesky_inverse(G, bp, b, round == 0 ? ref : std::vector<double>(b, 0.0), Rinv);
        if (!bad.empty()) {
          CB_TRY(randomize(k, bad));
          ok = false;
          break;
        }
        CB_TRY(combine(Vk, M, bp, Rinv, bp, false, Z, bp));
        CB_TRY(copy_cols(Vk, M, Z, bp, bp));
        if (with_w) {
          CB_TRY(combine(Wk, M, bp, Rinv, bp, false, Z, bp));
          CB_TRY(copy_cols(Wk, M, Z, bp, bp));
        }
      }
      if (ok) return CB_OK;
      if (with_w) CB_TRY(product(p));  // the replaced columns need their products again
    }
    CB_CHECK(false, CB_ERR_UNSUPPORTED, "multidimensional scaling: no independent basis block found");
  }
};

// order of |theta| descending, the positive value first at equal magnitude, then the lower index
std::vector<int> magnitude_order(const std::vector<double>& th) {
  std::vector<int> o(th.size());
  std::iota(o.begin(), o.end(), 0);
  std::stable_sort(o.begin(), o.end(), [&](int x, int y) {
    const double ax = std::fabs(th[x]), ay = std::fabs(th[y]);
    if (ax != ay) return ax > ay;
    return th[x] > th[y];
  });
  return o;
}

constexpr int kMaxRestarts = 500;
constexpr double kTol = 1e-7;  // the reference's float tolerance

// estimateEmbeddingDimensionEigengap (multidimensional_scaling.hpp:9-31) on fp32 values
size_t mds_eigengap_dim(const float* ev, size_t m, size_t max_dim) {
  float mn = std::numeric_limits<float>::infinity(), mx = -std::numeric_limits<float>::infinity();
  float best = -std::numeric_limits<float>::infinity();
  size_t ind = 0;
  for (size_t i = 0; i + 1 < m; i++) {
    const float d = ev[i] - ev[i + 1];
    if (d > best) {
      best = d;
      ind = i;
    }
    if (ev[i] < mn) mn = ev[i];
    if (ev[i] > mx) mx = ev[i];
  }
  if (ev[m - 1] < mn) mn = ev[m - 1];
  if (ev[m - 1] > mx) mx = ev[m - 1];
  if (mx - mn < std::numeric_limits<float>::epsilon()) return max_dim;
  return ind + 1;
}

}  // namespace

static int vectors_mds(cb_context* ctx, const cb_vectors* dist, size_t max_dim, int estimate_dim,
                       int distances_are_squared, float* evals, size_t* nev_out, size_t* dim_out, float* emb_host,
                       cb_vectors** emb_device) {
  CB_CHECK(ctx && dist && evals && nev_out && dim_out, CB_ERR_INVALID, "null argument");
  if (emb_device) *emb_device = nullptr;
  CB_CHECK(dist->ctx == ctx, CB_ERR_INVALID, "vector set belongs to another context");
  CB_CHECK(ctx->world == 1, CB_ERR_UNSUPPORTED, "multidimensional scaling runs on one GPU");
  const size_t n = dist->n;
  CB_CHECK((size_t)dist->D == n, CB_ERR_INVALID, "the distance matrix must be square (D == n)");
  CB_CHECK(n >= 2, CB_ERR_INVALID, "the distance matrix needs at least 2 rows");
  const size_t nev = estimate_dim ? std::min(max_dim + 1, n - 1) : max_dim;
  // Spectra's rule: 1 <= nev <= n - 1 (ncv = min(2 nev, n) > nev)
  CB_CHECK(nev >= 1 && nev <= n - 1, CB_ERR_INVALID, "number of eigenvalues out of [1, n - 1]");
  CB_CHECK(!estimate_dim || max_dim <= n - 1, CB_ERR_INVALID, "max_dim must be below n when the dimension is estimated");
  CB_CUDA(cudaSetDevice(ctx->device));
  *nev_out = nev;
  const float nanf = std::numeric_limits<float>::quiet_NaN();
  DeviceScope scope(ctx);
  Solver S(ctx, scope, dist->d_raw, n, !distances_are_squared);

  // means
  const int nchunks = (int)((n + kMeansCols - 1) / kMeansCols), nslabs = (int)((n + kMeansRows - 1) / kMeansRows);
  double *rowpart, *colpart, *sums, *d_g;
  CB_TRY(scope.alloc(&rowpart, (size_t)nchunks * n));
  CB_TRY(scope.alloc(&colpart, (size_t)nslabs * n));
  CB_TRY(scope.alloc(&sums, 2 * n));
  CB_TRY(scope.alloc(&S.rg, n));
  CB_TRY(scope.alloc(&S.cm, n));
  CB_TRY(scope.alloc(&d_g, 1));
  if (S.square)
    CB_TRY(launch(ctx, mds_means_kernel<true>, dim3((unsigned)nchunks, (unsigned)nslabs), kThreads, 0, S.dm, n,
                  rowpart, colpart));
  else
    CB_TRY(launch(ctx, mds_means_kernel<false>, dim3((unsigned)nchunks, (unsigned)nslabs), kThreads, 0, S.dm, n,
                  rowpart, colpart));
  CB_TRY(launch(ctx, mds_means_fold_kernel, grid_for(ctx, 2 * n, 256), 256, 0, rowpart, colpart, n, nchunks, nslabs,
                sums));
  CB_TRY(launch(ctx, mds_means_finish_kernel, 1, 1024, 0, sums, n, S.rg, S.cm, d_g));
  double g = 0.0;
  CB_CUDA(cudaMemcpyAsync(&g, d_g, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  CB_TRY(scope.free(rowpart));
  CB_TRY(scope.free(colpart));

  std::vector<double> lam(nev, std::numeric_limits<double>::quiet_NaN());
  std::vector<double> vecs;  // n x bp, the first nev columns the eigenvectors
  int rc = 1;
  if (!std::isfinite(g)) {  // a non-finite (squared) entry: every sum is non-finite
    rc = 0;
  } else {
    // basis: blocks of b >= nev + 2 columns, s blocks deep; the whole space at once when n <= 2 b
    S.b = (int)std::min<size_t>(n, ((nev + 2 + 7) / 8) * 8);
    if (n <= 2 * (size_t)S.b) {
      S.b = (int)n;
      S.s = 1;
    } else {
      S.s = (int)std::min<size_t>(4, n / (size_t)S.b);
    }
    S.bp = ((S.b + 7) / 8) * 8;
    S.M = S.s * S.bp;
    const int M = S.M, bp = S.bp, b = S.b;
    CB_TRY(scope.alloc(&S.V, n * (size_t)M));
    CB_TRY(scope.alloc(&S.W, n * (size_t)M));
    CB_TRY(scope.alloc(&S.Z, n * (size_t)bp));
    CB_TRY(scope.alloc(&S.Z2, n * (size_t)bp));
    CB_CUDA(cudaMemsetAsync(S.V, 0, n * (size_t)M * sizeof(double), ctx->stream));
    CB_CUDA(cudaMemsetAsync(S.W, 0, n * (size_t)M * sizeof(double), ctx->stream));
    CB_TRY(S.setup_product());
    std::vector<int> all((size_t)b);
    std::iota(all.begin(), all.end(), 0);
    CB_TRY(S.randomize(0, all));
    CB_TRY(S.orthonormalize(0, false));
    CB_TRY(S.product(0));
    // real columns of the padded basis
    std::vector<int> cols;
    for (int k = 0; k < S.s; k++)
      for (int j = 0; j < b; j++) cols.push_back(k * bp + j);
    const int m = (int)cols.size();
    const float eps32 = std::numeric_limits<float>::epsilon();
    const double eps23 = std::pow((double)eps32, 2.0 / 3.0);
    bool converged = false;
    std::vector<double> G, Hm((size_t)m * m), th((size_t)m), Y((size_t)m * m), sel;
    for (int it = 0; it < kMaxRestarts && !converged; it++) {
      for (int k = 1; k < S.s; k++) {  // Krylov block k from B times block k - 1
        CB_TRY(S.copy_cols(S.V + (size_t)k * bp, M, S.W + (size_t)(k - 1) * bp, M, bp));
        CB_TRY(S.orthonormalize(k, false));
        CB_TRY(S.product(k * bp));
      }
      // Rayleigh-Ritz: H = V^T B V (symmetrised)
      CB_TRY(S.gram(S.V, M, M, S.W, M, M, G));
      for (int x = 0; x < m; x++)
        for (int y = 0; y < m; y++)
          Hm[(size_t)x * m + y] =
              0.5 * (G[(size_t)cols[x] * M + cols[y]] + G[(size_t)cols[y] * M + cols[x]]);
      const int er = sym_eigen_f64(Hm.data(), m, th.data(), Y.data());
      CB_CHECK(er == 1, CB_ERR_UNSUPPORTED, "multidimensional scaling: the projected eigen-solve failed");
      const std::vector<int> ord = magnitude_order(th);
      // the b leading Ritz vectors as M x bp coefficients (padded rows / columns zero)
      sel.assign((size_t)M * bp, 0.0);
      std::vector<double> selt((size_t)M * bp, 0.0);  // Y diag(theta) for the residuals
      for (int j = 0; j < b; j++)
        for (int x = 0; x < m; x++) {
          sel[(size_t)cols[x] * bp + j] = Y[(size_t)x * m + ord[j]];
          selt[(size_t)cols[x] * bp + j] = -Y[(size_t)x * m + ord[j]] * th[ord[j]];
        }
      // residuals B v - theta v = W y - V y theta of the nev kept pairs
      CB_TRY(S.combine(S.W, M, M, sel, bp, false, S.Z, bp));
      CB_TRY(S.combine(S.V, M, M, selt, bp, true, S.Z, bp));
      CB_TRY(S.gram(S.Z, bp, bp, S.Z, bp, bp, G));
      const double th1 = std::fabs(th[ord[0]]);
      converged = true;
      for (size_t j = 0; j < nev; j++) {
        const double res = std::sqrt(std::max(0.0, G[j * bp + j]));
        converged = converged && res <= kTol * std::max(eps23 * th1, std::fabs(th[ord[j]]));
      }
      // restart from the b leading Ritz vectors and their products
      CB_TRY(S.combine(S.V, M, M, sel, bp, false, S.Z, bp));
      CB_TRY(S.combine(S.W, M, M, sel, bp, false, S.Z2, bp));
      CB_TRY(S.copy_cols(S.V, M, S.Z, bp, bp));
      CB_TRY(S.copy_cols(S.W, M, S.Z2, bp, bp));
      if (converged) {
        for (size_t j = 0; j < nev; j++) lam[j] = th[ord[j]];
        break;
      }
      CB_TRY(S.orthonormalize(0, true));
    }
    if (!converged) {
      std::fill(evals, evals + nev, nanf);
      CB_CHECK(false, CB_ERR_UNSUPPORTED, "multidimensional scaling: the eigen-solve did not converge");
    }
    vecs.resize(n * (size_t)bp);
    // Z (n x bp) still holds V Y: the Ritz vectors of the kept pairs in their order
    CB_CUDA(cudaMemcpyAsync(vecs.data(), S.Z, n * (size_t)bp * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
  }

  // clamp, estimate the dimension, embed
  for (size_t j = 0; j < nev; j++) evals[j] = rc == 1 ? (float)std::max(0.0, lam[j]) : nanf;
  const size_t dim = estimate_dim ? mds_eigengap_dim(evals, nev, max_dim) : max_dim;
  *dim_out = dim;
  std::vector<float> emb(n * dim, nanf);
  if (rc == 1) {
    const int bp = S.bp;
    for (size_t d = 0; d < dim; d++) {
      size_t big = 0;  // sign rule: the largest-magnitude component positive, the lowest index on ties
      for (size_t i = 1; i < n; i++)
        if (std::fabs(vecs[i * bp + d]) > std::fabs(vecs[big * bp + d])) big = i;
      const double sg = vecs[big * bp + d] < 0.0 ? -1.0 : 1.0;
      const double sl = std::sqrt((double)evals[d]);
      for (size_t i = 0; i < n; i++) emb[i * dim + d] = (float)(sl * (sg * vecs[i * bp + d]));
    }
  }
  if (emb_host) std::copy(emb.begin(), emb.end(), emb_host);
  if (emb_device) {
    cb_vectors* res = new cb_vectors(ctx, n, (int)dim);
    auto up = [&]() -> int {
      CB_TRY(res->mem.alloc(&res->d_raw, n * dim));
      CB_CUDA(cudaMemcpyAsync(res->d_raw, emb.data(), n * dim * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
      CB_CUDA(cudaStreamSynchronize(ctx->stream));
      return CB_OK;
    };
    const int urc = up();
    if (urc != CB_OK) {
      delete res;
      return urc;
    }
    *emb_device = res;
  }
  return rc;
}

extern "C" {

int cb_vectors_mds(cb_context* ctx, const cb_vectors* dist, size_t max_dim, int estimate_dim,
                   int distances_are_squared, float* eigenvalues, size_t* nev, size_t* dim, float* embedded_host,
                   cb_vectors** embedded_device) {
  return vectors_mds(ctx, dist, max_dim, estimate_dim, distances_are_squared, eigenvalues, nev, dim, embedded_host,
                     embedded_device);
}

}  // extern "C"
