// Depth-image and RGB-D <-> point-cloud conversions (core/image_point_cloud_conversions.hpp) under the contract of
// DESIGN §4.20: fp32, one rounding per operation (no FMA), the reference's per-branch association, an order-preserving
// compaction and a deterministic z-buffer.
//
// Image -> cloud: one kernel over 32 x 8 pixel tiles back-projects each pixel, decides its validity and, for the
// ...Normals variants, computes its normal from a one-pixel halo of back-projected points in shared memory. With
// keep_invalid that kernel writes every pixel (1 launch). Otherwise it runs twice around exclusive_scan_u32: a counting
// pass writes one keep flag per pixel, the scan turns the flags into output offsets, and a writing pass recomputes the
// pixel (reading the 2-4 B raw value again is cheaper than storing 24-36 B of temporaries) and scatters the kept ones
// in ascending pixel order (1 + 3 + 1 = 5 launches).
//
// Cloud -> image: a point pass atomicMin()s (key << 32 | point index) into a 64-bit word per pixel, the key being the
// raw depth (depth / RGB-D) or the bits of the metric z (index map), which order like the values for positive floats;
// a pixel pass writes the winner's raw depth, colour or index (2 launches). This is the reference's serial result:
// smallest key, lowest index on ties, the colour of the winner.
#include "cb_internal.hpp"
#include "launch.cuh"
#include "projection.hpp"
#include <cmath>
#include <cstring>

using namespace cb;

namespace {

constexpr int kTileW = 32, kTileH = 8, kThreads = kTileW * kTileH;
constexpr int kHaloW = kTileW + 2, kHaloH = kTileH + 2;
constexpr unsigned long long kEmpty = ~0ull;

// ---- host restatement of the fixed-order fp32 operations (volatile: each result is rounded once, never fused) ----
float rmul(float a, float b) {
  volatile float r = a * b;
  return r;
}
float radd(float a, float b) {
  volatile float r = a + b;
  return r;
}
float rsub(float a, float b) {
  volatile float r = a - b;
  return r;
}
float rdiv(float a, float b) {
  volatile float r = a / b;
  return r;
}
// Eigen's dot of two 3-vectors: (a0 b0 + a1 b1) + a2 b2
float rdot(float a0, float a1, float a2, float b0, float b1, float b2) {
  return radd(radd(rmul(a0, b0), rmul(a1, b1)), rmul(a2, b2));
}

// intrinsics.inverse() for a fixed 3 x 3 float matrix as Eigen 3.4 computes it (compute_inverse<..., 3>): the cofactors
// C(i, j) = m(i1, j1) m(i2, j2) - m(i1, j2) m(i2, j1) (i1 = i + 1, i2 = i + 2 mod 3), det = (C00 m00 + C10 m10) + C20 m20,
// invdet = 1 / det, inverse(i, j) = C(j, i) * invdet. K and Ki are row-major.
void inverse3(const float* K, float* Ki) {
  auto m = [&](int r, int c) { return K[3 * r + c]; };
  auto cof = [&](int i, int j) {
    const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
    return rsub(rmul(m(i1, j1), m(i2, j2)), rmul(m(i1, j2), m(i2, j1)));
  };
  const float det = rdot(cof(0, 0), cof(1, 0), cof(2, 0), m(0, 0), m(1, 0), m(2, 0));
  const float invdet = rdiv(1.0f, det);
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) Ki[3 * i + j] = rmul(cof(j, i), invdet);
}

// ---- device ------------------------------------------------------------------------------------------------------
struct BackProject {
  const void* depth;
  const uint8_t* rgb;  // or nullptr
  uint32_t w, h;
  int truncated;
  float inv_scale, max_depth;
  float A[9];   // row-major: p = A v (K^-1, or t 1^T + R K^-1 for the keep_invalid points-only extrinsics branch)
  int post;     // output points p' = R p + t and normals R n
  float R[9], t[3];
  float* pts;   // 3 floats per output point
  float* nrm;   // or nullptr
  float* col;   // or nullptr
  uint32_t* flag;          // counting pass: one keep flag per pixel
  const uint32_t* offset;  // writing pass: output slot of each kept pixel
};

__device__ __forceinline__ float dot3(const float* a, float b0, float b1, float b2) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a[0], b0), __fmul_rn(a[1], b1)), __fmul_rn(a[2], b2));
}

template <class Raw>
__device__ __forceinline__ float3 back_project(const BackProject& P, uint32_t x, uint32_t y) {
  const Raw raw = static_cast<const Raw*>(P.depth)[(size_t)y * P.w + x];
  float z = __fmul_rn(P.inv_scale, (float)raw);
  if (P.truncated) z = z < P.max_depth ? z : 0.0f;
  const float v0 = __fmul_rn(z, (float)x), v1 = __fmul_rn(z, (float)y);
  return make_float3(dot3(P.A, v0, v1, z), dot3(P.A + 3, v0, v1, z), dot3(P.A + 6, v0, v1, z));
}

// (dn - up) x (rt - lf), normalised as Eigen's normalized(): divided by sqrt((x^2 + y^2) + z^2) when that is > 0
__device__ __forceinline__ float3 pixel_normal(float3 up, float3 dn, float3 lf, float3 rt) {
  const float ax = __fsub_rn(dn.x, up.x), ay = __fsub_rn(dn.y, up.y), az = __fsub_rn(dn.z, up.z);
  const float bx = __fsub_rn(rt.x, lf.x), by = __fsub_rn(rt.y, lf.y), bz = __fsub_rn(rt.z, lf.z);
  float cx = __fsub_rn(__fmul_rn(ay, bz), __fmul_rn(az, by));
  float cy = __fsub_rn(__fmul_rn(az, bx), __fmul_rn(ax, bz));
  float cz = __fsub_rn(__fmul_rn(ax, by), __fmul_rn(ay, bx));
  const float s = __fadd_rn(__fadd_rn(__fmul_rn(cx, cx), __fmul_rn(cy, cy)), __fmul_rn(cz, cz));
  if (s > 0.0f) {
    const float r = __fsqrt_rn(s);
    cx = __fdiv_rn(cx, r);
    cy = __fdiv_rn(cy, r);
    cz = __fdiv_rn(cz, r);
  }
  return make_float3(cx, cy, cz);
}

enum Pass { kKeepAll = 0, kCount = 1, kWrite = 2 };

// One block per 32 x 8 tile of the image (tiles numbered row-major, tiles_x per row).
template <class Raw, bool kNormals, int kPass>
__global__ void __launch_bounds__(kThreads) depth_points_kernel(const BackProject P, uint32_t tiles_x) {
  __shared__ float3 tile[kNormals ? kHaloH * kHaloW : 1];
  const uint32_t x0 = (blockIdx.x % tiles_x) * kTileW, y0 = (blockIdx.x / tiles_x) * kTileH;
  const uint32_t lx = threadIdx.x % kTileW, ly = threadIdx.x / kTileW;
  const uint32_t x = x0 + lx, y = y0 + ly;
  const bool inside = x < P.w && y < P.h;
  const float qnan = __int_as_float(0x7fffffff);
  float3 p, n = make_float3(qnan, qnan, qnan);
  if (kNormals) {
    for (int i = threadIdx.x; i < kHaloH * kHaloW; i += kThreads) {
      const long long hx = (long long)x0 - 1 + i % kHaloW, hy = (long long)y0 - 1 + i / kHaloW;
      float3 q = make_float3(0.0f, 0.0f, 0.0f);  // outside the image: only read for pixels that get no normal
      if (hx >= 0 && hy >= 0 && hx < P.w && hy < P.h) q = back_project<Raw>(P, (uint32_t)hx, (uint32_t)hy);
      tile[i] = q;
    }
    __syncthreads();
    if (!inside) return;
    const int c = (ly + 1) * kHaloW + lx + 1;
    p = tile[c];
    if (x >= 1 && y >= 1 && x + 1 < P.w && y + 1 < P.h) {
      const float3 up = tile[c - kHaloW], dn = tile[c + kHaloW], lf = tile[c - 1], rt = tile[c + 1];
      if (p.z > 0.0f && rt.z > 0.0f && lf.z > 0.0f && dn.z > 0.0f && up.z > 0.0f) n = pixel_normal(up, dn, lf, rt);
    }
  } else {
    if (!inside) return;
    p = back_project<Raw>(P, x, y);
  }
  const size_t k = (size_t)y * P.w + x;
  const bool keep = kNormals ? !isnan(n.x) : p.z > 0.0f;
  if (kPass == kCount) {
    P.flag[k] = keep ? 1u : 0u;
    return;
  }
  size_t o = k;
  if (kPass == kWrite) {
    if (!keep) return;
    o = P.offset[k];
  }
  if (P.post) {
    p = make_float3(__fadd_rn(dot3(P.R, p.x, p.y, p.z), P.t[0]), __fadd_rn(dot3(P.R + 3, p.x, p.y, p.z), P.t[1]),
                    __fadd_rn(dot3(P.R + 6, p.x, p.y, p.z), P.t[2]));
    if (kNormals) n = make_float3(dot3(P.R, n.x, n.y, n.z), dot3(P.R + 3, n.x, n.y, n.z), dot3(P.R + 6, n.x, n.y, n.z));
  }
  P.pts[3 * o] = p.x;
  P.pts[3 * o + 1] = p.y;
  P.pts[3 * o + 2] = p.z;
  if (kNormals && P.nrm) {
    P.nrm[3 * o] = n.x;
    P.nrm[3 * o + 1] = n.y;
    P.nrm[3 * o + 2] = n.z;
  }
  if (P.col) {
    const float mult = 1.0f / 255.0f;
    for (int c = 0; c < 3; c++) P.col[3 * o + c] = __fmul_rn(mult, (float)P.rgb[3 * k + c]);
  }
}

enum RenderMode { kDepthU16 = 0, kDepthF32 = 1, kIndexMap = 2 };

struct Render {
  const float* pts;
  uint32_t n;
  int mode;  // RenderMode
  int truncated;
  float scale, max_depth;
  Projection prj;  // intrinsics, extrinsics.inverse(), image size (projection.hpp)
  unsigned long long* keys;  // w * h, kEmpty on entry
};

__global__ void __launch_bounds__(256) render_keys_kernel(const Render P) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < P.n; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t px, py;
    float q2;
    if (!project_pixel(P.prj, P.pts[3 * i], P.pts[3 * i + 1], P.pts[3 * i + 2], px, py, q2)) continue;
    uint32_t key;
    if (P.mode == kIndexMap) {
      key = __float_as_uint(q2);
    } else {
      if (P.truncated && !(q2 < P.max_depth)) continue;
      const float v = __fmul_rn(P.scale, q2);
      if (P.mode == kDepthU16) {
        if (!(v >= 0.0f && v < 65536.0f)) continue;  // does not fit an unsigned short: skipped
        key = __float2uint_rz(v);
      } else {
        if (!(v > 0.0f)) continue;
        key = __float_as_uint(v);
      }
      if (key == 0) continue;  // a raw depth of 0 never writes
    }
    atomicMin(&P.keys[(size_t)py * P.prj.w + px], ((unsigned long long)key << 32) | i);
  }
}

__device__ __forceinline__ uint8_t color_byte(float c) {
  const float v = __fmul_rn(255.0f, c);
  if (!(v > 0.0f)) return 0;  // NaN and v <= 0 saturate to 0
  if (v >= 255.0f) return 255;
  return (uint8_t)__float2uint_rz(v);
}

// mode kIndexMap: keys becomes the index map in place
__global__ void __launch_bounds__(256) render_write_kernel(unsigned long long* keys, size_t npix, int mode,
                                                           const float* col, void* depth, uint8_t* rgb,
                                                           unsigned long long index_offset) {
  for (size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x; k < npix; k += (size_t)gridDim.x * blockDim.x) {
    const unsigned long long key = keys[k];
    const bool empty = key == kEmpty;
    const uint32_t hi = (uint32_t)(key >> 32), idx = (uint32_t)key;
    if (mode == kIndexMap) {
      keys[k] = empty ? kEmpty : (unsigned long long)idx + index_offset;
      continue;
    }
    if (mode == kDepthU16)
      static_cast<uint16_t*>(depth)[k] = empty ? (uint16_t)0 : (uint16_t)hi;
    else
      static_cast<float*>(depth)[k] = empty ? 0.0f : __uint_as_float(hi);
    if (col)
      for (int c = 0; c < 3; c++) rgb[3 * k + c] = empty ? (uint8_t)0 : color_byte(col[3 * (size_t)idx + c]);
  }
}

// ---- host ----------------------------------------------------------------------------------------------------------
// 1: device (or managed) memory of the context's device, 0: host memory, -1: device memory of another device
int memory_kind(const cb_context* ctx, const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  if (a.type == cudaMemoryTypeManaged) return 1;
  if (a.type != cudaMemoryTypeDevice) return 0;
  return a.device == ctx->device ? 1 : -1;
}

int check_converter(const cb_depth_converter* conv) {
  CB_CHECK(conv, CB_ERR_INVALID, "null converter");
  CB_CHECK(conv->raw_type == CB_DEPTH_U16 || conv->raw_type == CB_DEPTH_F32, CB_ERR_INVALID, "unknown raw depth type");
  CB_CHECK(std::isfinite(conv->scale) && conv->scale != 0.0f, CB_ERR_INVALID, "scale must be finite and nonzero");
  return CB_OK;
}

int check_image(size_t w, size_t h) {
  CB_CHECK(w > 0 && h > 0, CB_ERR_INVALID, "empty image");
  CB_CHECK(w < (1ull << 32) && h < (1ull << 32) && (unsigned __int128)w * h < ((unsigned __int128)1 << 32),
           CB_ERR_UNSUPPORTED, "images of >= 2^32 pixels are not supported");
  return CB_OK;
}

// A device copy of n elements of T at p (the caller's buffer itself when it is device memory).
template <class T>
int device_view(cb_context* ctx, DeviceScope& scope, const T* p, size_t n, const T** out) {
  const int kind = memory_kind(ctx, p);
  CB_CHECK(kind >= 0, CB_ERR_INVALID, "image in the memory of another device");
  if (kind == 1) {
    *out = p;
    return CB_OK;
  }
  T* d = nullptr;
  CB_TRY(scope.alloc(&d, n));
  CB_CUDA(cudaMemcpyAsync(d, p, n * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
  *out = d;
  return CB_OK;
}

template <class Raw, bool kNormals, int kPass>
int launch_depth_points(cb_context* ctx, const BackProject& P) {
  const uint32_t tiles_x = (P.w + kTileW - 1) / kTileW, tiles_y = (P.h + kTileH - 1) / kTileH;
  return launch(ctx, depth_points_kernel<Raw, kNormals, kPass>, dim3((unsigned)((size_t)tiles_x * tiles_y)),
                dim3(kThreads), 0, P, tiles_x);
}

template <int kPass>
int launch_depth_points(cb_context* ctx, const BackProject& P, bool f32, bool normals) {
  if (f32) return normals ? launch_depth_points<float, true, kPass>(ctx, P) : launch_depth_points<float, false, kPass>(ctx, P);
  return normals ? launch_depth_points<uint16_t, true, kPass>(ctx, P) : launch_depth_points<uint16_t, false, kPass>(ctx, P);
}

int depth_to_points(cb_context* ctx, const void* depth, const unsigned char* rgb, size_t w, size_t h,
                    const cb_depth_converter* conv, const float* K, const float* extr, bool normals, bool keep_invalid,
                    float* h_pts, float* h_nrm, float* h_col, size_t* count, cb_cloud** out_device) {
  const size_t npix = w * h;
  const bool f32 = conv->raw_type == CB_DEPTH_F32;
  DeviceScope scope(ctx);
  BackProject P;
  std::memset(&P, 0, sizeof(P));
  if (f32) {
    const float* d = nullptr;
    CB_TRY(device_view(ctx, scope, static_cast<const float*>(depth), npix, &d));
    P.depth = d;
  } else {
    const uint16_t* d = nullptr;
    CB_TRY(device_view(ctx, scope, static_cast<const uint16_t*>(depth), npix, &d));
    P.depth = d;
  }
  if (h_col) CB_TRY(device_view(ctx, scope, rgb, 3 * npix, &P.rgb));
  P.w = (uint32_t)w;
  P.h = (uint32_t)h;
  P.truncated = conv->truncated ? 1 : 0;
  P.inv_scale = rdiv(1.0f, conv->scale);
  P.max_depth = conv->max_depth;
  float Ki[9];
  inverse3(K, Ki);
  std::memcpy(P.A, Ki, sizeof(Ki));
  if (extr) {
    for (int i = 0; i < 3; i++) {
      for (int j = 0; j < 3; j++) P.R[3 * i + j] = extr[4 * i + j];
      P.t[i] = extr[4 * i + 3];
    }
    if (keep_invalid && !normals) {
      // (extrinsics * intrinsics_inv) * v: an isometry times a 3 x 3 matrix takes its columns as three points, so the
      // product is R K^-1 with t added to every column, and v is then multiplied by that matrix
      for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++)
          P.A[3 * i + j] = radd(P.t[i], rdot(P.R[3 * i], P.R[3 * i + 1], P.R[3 * i + 2], Ki[j], Ki[3 + j], Ki[6 + j]));
    } else {
      P.post = 1;  // extrinsics * p (and extrinsics.linear() * n) after the back-projection
    }
  }
  size_t m = npix;
  if (!keep_invalid) {
    uint32_t* d_flag = nullptr;
    CB_TRY(scope.alloc(&d_flag, npix + 2));
    CB_CUDA(cudaMemsetAsync(d_flag + npix, 0, 2 * sizeof(uint32_t), ctx->stream));
    P.flag = d_flag;
    CB_TRY(launch_depth_points<kCount>(ctx, P, f32, normals));
    CB_TRY(exclusive_scan_u32(ctx, d_flag, npix + 1, 0u));
    uint32_t kept = 0;
    CB_CUDA(cudaMemcpyAsync(&kept, d_flag + npix, sizeof(kept), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    m = kept;
    P.offset = d_flag;
    P.flag = nullptr;
  }
  cb_cloud* c = nullptr;
  if (out_device) {
    CB_CHECK(m < (1ull << 31), CB_ERR_UNSUPPORTED, "clouds of >= 2^31 points are not supported");
    c = new cb_cloud(ctx, m, 0);
    int rc = c->mem.alloc(&c->d_raw, 3 * m);
    if (rc == CB_OK && normals) rc = c->mem.alloc(&c->d_raw_nrm, 3 * m);
    if (rc != CB_OK) {
      delete c;
      return rc;
    }
    P.pts = c->d_raw;
    P.nrm = c->d_raw_nrm;
  }
  auto fill = [&]() -> int {
    if (!P.pts) CB_TRY(scope.alloc(&P.pts, 3 * m));
    if (normals && !P.nrm && h_nrm) CB_TRY(scope.alloc(&P.nrm, 3 * m));
    if (h_col) CB_TRY(scope.alloc(&P.col, 3 * m));
    if (m) {
      if (keep_invalid)
        CB_TRY(launch_depth_points<kKeepAll>(ctx, P, f32, normals));
      else
        CB_TRY(launch_depth_points<kWrite>(ctx, P, f32, normals));
    }
    const size_t bytes = 3 * m * sizeof(float);
    if (h_pts && m) CB_CUDA(cudaMemcpyAsync(h_pts, P.pts, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    if (h_nrm && m) CB_CUDA(cudaMemcpyAsync(h_nrm, P.nrm, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    if (h_col && m) CB_CUDA(cudaMemcpyAsync(h_col, P.col, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    return CB_OK;
  };
  const int rc = fill();
  if (rc != CB_OK) {
    delete c;
    return rc;
  }
  *count = m;
  if (out_device) *out_device = c;
  return CB_OK;
}

// keys (w * h) = the z-buffer of P.pts: (key << 32 | index) of each pixel's winner, kEmpty where no point lands
int zbuffer(cb_context* ctx, const Render& P) {
  CB_CUDA(cudaMemsetAsync(P.keys, 0xff, (size_t)P.prj.w * P.prj.h * sizeof(unsigned long long), ctx->stream));
  return launch(ctx, render_keys_kernel, grid_for(ctx, P.n, 256), 256, 0, P);
}

int render(cb_context* ctx, const float* xyz, const cb_cloud* cloud, size_t n, const float* colors, const float* K,
           const float* extr, int mode, const cb_depth_converter* conv, size_t w, size_t h, void* depth, uint8_t* rgb,
           uint64_t* index_map) {
  CB_CHECK(K && (xyz == nullptr) != (cloud == nullptr), CB_ERR_INVALID, "need K and exactly one of xyz and cloud");
  CB_TRY(check_image(w, h));
  if (cloud) {
    CB_CHECK(cloud->ctx == ctx, CB_ERR_INVALID, "cloud of another context");
    n = cloud->n;
  }
  CB_CHECK(n < (1ull << 32), CB_ERR_UNSUPPORTED, "point sets of >= 2^32 points are not supported");
  CB_CUDA(cudaSetDevice(ctx->device));
  const size_t npix = w * h;
  DeviceScope scope(ctx);
  Render P;
  std::memset(&P, 0, sizeof(P));
  P.n = (uint32_t)n;
  P.mode = mode;
  if (conv) {
    P.truncated = conv->truncated ? 1 : 0;
    P.scale = conv->scale;
    P.max_depth = conv->max_depth;
  }
  P.prj = make_projection(K, extr, (uint32_t)w, (uint32_t)h);
  if (cloud) {
    P.pts = cloud->d_raw;
  } else if (n) {
    float* d = nullptr;
    CB_TRY(scope.alloc(&d, 3 * n));
    CB_CUDA(cudaMemcpyAsync(d, xyz, 3 * n * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    P.pts = d;
  }
  float* d_col = nullptr;
  if (colors) {
    CB_TRY(scope.alloc(&d_col, 3 * n));
    if (n) CB_CUDA(cudaMemcpyAsync(d_col, colors, 3 * n * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  }
  CB_TRY(scope.alloc(&P.keys, npix));
  CB_TRY(zbuffer(ctx, P));
  void* d_depth = nullptr;
  uint8_t* d_rgb = nullptr;
  const size_t depth_bytes = npix * (mode == kDepthU16 ? sizeof(uint16_t) : sizeof(float));
  if (mode != kIndexMap) {
    uint8_t* d = nullptr;
    CB_TRY(scope.alloc(&d, depth_bytes));
    d_depth = d;
  }
  if (colors) CB_TRY(scope.alloc(&d_rgb, 3 * npix));
  CB_TRY(launch(ctx, render_write_kernel, grid_for(ctx, npix, 256), 256, 0, P.keys, npix, mode, (const float*)d_col,
                d_depth, d_rgb, (unsigned long long)(cloud ? cloud->index_offset : 0)));
  if (mode == kIndexMap)
    CB_CUDA(cudaMemcpyAsync(index_map, P.keys, npix * sizeof(uint64_t), cudaMemcpyDeviceToHost, ctx->stream));
  else
    CB_CUDA(cudaMemcpyAsync(depth, d_depth, depth_bytes, cudaMemcpyDeviceToHost, ctx->stream));
  if (colors) CB_CUDA(cudaMemcpyAsync(rgb, d_rgb, 3 * npix, cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  return CB_OK;
}

}  // namespace

namespace cb {
int index_map_keys(cb_context* ctx, const float* d_pts, size_t n, const Projection& prj, unsigned long long* keys) {
  Render P;
  std::memset(&P, 0, sizeof(P));
  P.pts = d_pts;
  P.n = (uint32_t)n;
  P.mode = kIndexMap;
  P.prj = prj;
  P.keys = keys;
  return zbuffer(ctx, P);
}
}  // namespace cb

int cb_depth_image_to_points(cb_context* ctx, const void* depth, const unsigned char* rgb, size_t w, size_t h,
                             const cb_depth_converter* conv, const float* K, const float* extrinsics, int want_normals,
                             int keep_invalid, float* points, float* normals, float* colors, size_t* count,
                             cb_cloud** out_device) {
  CB_CHECK(ctx && depth && K && count, CB_ERR_INVALID, "null argument");
  CB_TRY(check_converter(conv));
  CB_TRY(check_image(w, h));
  CB_CHECK(!colors || rgb, CB_ERR_INVALID, "colors need an rgb image");
  CB_CHECK(!normals || want_normals, CB_ERR_INVALID, "normals need want_normals");
  CB_CUDA(cudaSetDevice(ctx->device));
  if (out_device) *out_device = nullptr;
  return depth_to_points(ctx, depth, rgb, w, h, conv, K, extrinsics, want_normals != 0, keep_invalid != 0, points,
                         normals, colors, count, out_device);
}

int cb_points_to_depth_image(cb_context* ctx, const float* xyz, const cb_cloud* cloud, size_t n, const float* colors,
                             const float* K, const float* extrinsics, const cb_depth_converter* conv, size_t w,
                             size_t h, void* depth, unsigned char* rgb) {
  CB_CHECK(ctx && depth, CB_ERR_INVALID, "null argument");
  CB_TRY(check_converter(conv));
  CB_CHECK((colors == nullptr) == (rgb == nullptr), CB_ERR_INVALID, "colors and rgb go together");
  return render(ctx, xyz, cloud, n, colors, K, extrinsics, conv->raw_type == CB_DEPTH_U16 ? kDepthU16 : kDepthF32,
                conv, w, h, depth, rgb, nullptr);
}

int cb_points_to_index_map(cb_context* ctx, const float* xyz, const cb_cloud* cloud, size_t n, const float* K,
                           const float* extrinsics, size_t w, size_t h, uint64_t* index_map) {
  CB_CHECK(ctx && index_map, CB_ERR_INVALID, "null argument");
  return render(ctx, xyz, cloud, n, nullptr, K, extrinsics, kIndexMap, nullptr, w, h, nullptr, nullptr, index_map);
}
