// C ABI: context, clouds, nearest neighbour, rigid ICP (product code).
#include "cb_internal.hpp"
#include "feature_rule.hpp"
#include "feature_search.cuh"
#include "icp_kernels.cuh"
#include "stats_kernels.cuh"
#include "host_solve.hpp"
#include "icp_object.hpp"
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <cfloat>
#include <cmath>
#include <algorithm>
#include <vector>
#include <string>

namespace cb {

static thread_local std::string g_err;

void set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
}

int get_reduce_scratch(cb_context* ctx, int blocks, int nv, ReduceScratch* out) {
  const size_t groups = ((size_t)blocks + kReduceGroup - 1) / kReduceGroup;
  const size_t need = ((size_t)blocks + groups) * (size_t)nv;
  if (ctx->partials_cap < need) {
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    CB_TRY(ctx->mem.free(ctx->d_partials));
    const size_t cap = std::max<size_t>(need, (size_t)8192 * 32);
    CB_TRY(ctx->mem.alloc(&ctx->d_partials, cap));
    ctx->partials_cap = cap;
  }
  if (ctx->counter_cap < groups + 1) {
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    CB_TRY(ctx->mem.free(ctx->d_counter));
    const size_t cap = std::max<size_t>(groups + 1, 4096);
    CB_TRY(ctx->mem.alloc(&ctx->d_counter, cap));
    CB_CUDA(cudaMemsetAsync(ctx->d_counter, 0, cap * sizeof(unsigned int), ctx->stream));
    ctx->counter_cap = cap;
  }
  out->partials = ctx->d_partials;
  out->gpartials = ctx->d_partials + (size_t)blocks * nv;
  out->counters = ctx->d_counter;
  out->result = ctx->d_result;
  std::memset(&out->ex, 0, sizeof(out->ex));  // fused exchange off unless the caller arms it
  return CB_OK;
}

// ---- fused exchange: tables, arming, host wait -------------------------------------------------------
static inline unsigned long long* xchg_flags(void* base) { return reinterpret_cast<unsigned long long*>(base); }
static inline double* xchg_vals(void* base) {
  return reinterpret_cast<double*>(reinterpret_cast<char*>(base) + kXchgFlagBytes);
}

// (re)build the two device pointer tables from ctx->peer_xchg[0..world)
static int upload_peer_tables(cb_context* ctx) {
  double* hv[kMaxRanks];
  unsigned long long* hf[kMaxRanks];
  for (int p = 0; p < kMaxRanks; ++p) {
    void* base = (p < ctx->world && ctx->peer_xchg[p]) ? ctx->peer_xchg[p] : ctx->d_xchg;
    hv[p] = xchg_vals(base);
    hf[p] = xchg_flags(base);
  }
  CB_CUDA(cudaMemcpyAsync(ctx->d_peer_vals, hv, sizeof(hv), cudaMemcpyHostToDevice, ctx->stream));
  CB_CUDA(cudaMemcpyAsync(ctx->d_peer_flags, hf, sizeof(hf), cudaMemcpyHostToDevice, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  return CB_OK;
}

static int setup_exchange(cb_context* ctx) {
  CB_CUDA(cudaMalloc(&ctx->d_xchg, kXchgBytes));  // not from ctx->mem: CUDA IPC cannot export pool memory
  CB_CUDA(cudaMemset(ctx->d_xchg, 0, kXchgBytes));
  CB_TRY(ctx->mem.alloc(&ctx->d_peer_vals, kMaxRanks));
  CB_TRY(ctx->mem.alloc(&ctx->d_peer_flags, kMaxRanks));
  CB_TRY(ctx->mem.alloc_host(&ctx->h_sync, 64 + 4 * 64, cudaHostAllocMapped));
  std::memset(ctx->h_sync, 0, (64 + 4 * 64) * sizeof(unsigned long long));
  ctx->peer_xchg[0] = ctx->d_xchg;
  CB_TRY(upload_peer_tables(ctx));
  ctx->ex_ready = true;  // world == 1: no peers, host mailbox only
  return CB_OK;
}

// Bound of the in-kernel wait for the peers' rows (reduce.cuh, exchange_rows): CB_EXCHANGE_TIMEOUT_MS, default 20 s.
unsigned long long exchange_timeout_ns() {
  static const unsigned long long ns = [] {
    const char* e = getenv("CB_EXCHANGE_TIMEOUT_MS");
    const double ms = e ? atof(e) : 20000.0;
    return ms > 0 ? (unsigned long long)(ms * 1e6) : 0ull;
  }();
  return ns;
}

bool exchange_available(const cb_context* ctx) {
  static const bool disabled = getenv("CB_NO_FUSED_EXCHANGE") != nullptr;  // A/B switch for measurements
  return ctx->ex_ready && !disabled;
}

bool arm_exchange(cb_context* ctx, Exchange* ex) {
  if (!exchange_available(ctx)) return false;
  ex->enabled = 1;
  ex->rank = ctx->rank;
  ex->world = ctx->world;
  ex->seq = ++ctx->seq;
  ex->peer_vals = ctx->d_peer_vals;
  ex->peer_flags = ctx->d_peer_flags;
  ex->host_flag = ctx->h_sync;  // mapped pinned memory: same address on host and device (UVA)
  ex->host_vals = reinterpret_cast<double*>(ctx->h_sync + 8);
  // CB_TRACE_EXCHANGE=1: %globaltimer stamps of the last 64 passes in the mapped mailbox page
  static const bool trace = getenv("CB_TRACE_EXCHANGE") != nullptr;
  ex->trace = trace ? ctx->h_sync + 64 + 4 * (ctx->seq % 64) : nullptr;
  ex->timeout_ns = exchange_timeout_ns();
  return true;
}

int wait_exchange(cb_context* ctx, int count, double* out) {
  volatile unsigned long long* flag = ctx->h_sync;
  const unsigned long long want = ctx->seq;
  unsigned long long spins = 0;
  while (*flag != want) {
    if (*flag == (want | (1ull << 63))) {  // the kernel gave up waiting for a peer's row (reduce.cuh, exchange_rows)
      set_error("fused exchange: a peer rank did not deliver its row of pass %llu in time (rank %d of %d)", want,
                ctx->rank, ctx->world);
      ctx->ex_ready = false;
      return CB_ERR_NCCL;
    }
    if ((++spins & 0x3ffffull) == 0) {  // every ~0.3 ms: make sure the stream has not faulted or finished without us
      cudaError_t q = cudaStreamQuery(ctx->stream);
      if (q != cudaSuccess && q != cudaErrorNotReady) {
        set_error("kernel failed while waiting for the fused exchange: %s", cudaGetErrorString(q));
        return CB_ERR_CUDA;
      }
      if (q == cudaSuccess && *flag != want) {
        set_error("fused exchange: the pass finished without publishing its result");
        return CB_ERR_CUDA;
      }
    }
  }
  std::atomic_thread_fence(std::memory_order_acquire);
  const volatile double* v = reinterpret_cast<const volatile double*>(ctx->h_sync + 8);
  for (int i = 0; i < count; i++) out[i] = v[i];
  return CB_OK;
}

int fetch_result(cb_context* ctx, int count, bool allreduce, double* out) {
  if (allreduce && ctx->world > 1) CB_TRY(nccl_allreduce_sum_f64(ctx, ctx->d_result, (size_t)count));
  CB_CUDA(cudaMemcpyAsync(ctx->h_result, ctx->d_result, count * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  std::memcpy(out, ctx->h_result, count * sizeof(double));
  return CB_OK;
}

static Rigid to_rigid(const float* T12) { return rigid_from_t12(T12); }

}  // namespace cb

using namespace cb;

extern "C" {

const char* cb_last_error(void) { return cb::g_err.c_str(); }
const char* cb_version(void) { return "cilantro_b200 0.1 (sm_90a)"; }

// ---- context ------------------------------------------------------------------------------------
static int context_init(cb_context* ctx) {
  cudaDeviceProp prop;
  CB_CUDA(cudaGetDeviceProperties(&prop, ctx->device));
  ctx->sm_count = prop.multiProcessorCount;
  ctx->l2_bytes = (size_t)prop.l2CacheSize;
  ctx->hbm_bytes = prop.totalGlobalMem;
  snprintf(ctx->name, sizeof(ctx->name), "%s", prop.name);
  CB_CUDA(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
  {
    // All cloud / index / scratch buffers come from the stream-ordered pool. Keep freed memory in the
    // pool (default: returned to the OS at every synchronise, which made repeated cloud creation pay
    // page allocation again each time: large outliers in the end-to-end call).
    cudaMemPool_t pool;
    CB_CUDA(cudaDeviceGetDefaultMemPool(&pool, ctx->device));
    uint64_t keep = UINT64_MAX;
    CB_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
  }
  CB_TRY(ctx->mem.alloc(&ctx->d_result, 64));
  CB_CUDA(cudaMemsetAsync(ctx->d_result, 0, 64 * sizeof(double), ctx->stream));
  CB_TRY(ctx->mem.alloc_host(&ctx->h_result, 64));
  return setup_exchange(ctx);
}

int cb_context_create(int device, cb_context** out) {
  CB_CHECK(out, CB_ERR_INVALID, "out is null");
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count <= 0) {
    set_error("no CUDA device available (%s); cilantro_b200 has no CPU fallback",
              e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    return CB_ERR_NO_DEVICE;
  }
  CB_CHECK(device >= 0 && device < count, CB_ERR_INVALID, "device ordinal out of range");
  CB_CUDA(cudaSetDevice(device));
  cb_context* ctx = new cb_context;
  ctx->device = device;
  const int rc = context_init(ctx);
  if (rc != CB_OK) {
    cb_context_destroy(ctx);  // also destroys the stream and the exchange region
    return rc;
  }
  *out = ctx;
  return CB_OK;
}

void cb_context_destroy(cb_context* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  nccl_destroy(ctx);
  for (int p = 0; p < kMaxRanks; ++p)
    if (ctx->peer_xchg[p] && ctx->peer_xchg[p] != ctx->d_xchg) cudaIpcCloseMemHandle(ctx->peer_xchg[p]);
  if (ctx->d_xchg) cudaFree(ctx->d_xchg);
  if (ctx->d_flush) cudaFree(ctx->d_flush);
  const cudaStream_t stream = ctx->stream, copy_stream = ctx->copy_stream;
  delete ctx;  // ctx->mem frees its buffers on the stream, so the streams go after it
  if (copy_stream) cudaStreamDestroy(copy_stream);
  if (stream) cudaStreamDestroy(stream);
}

int cb_context_synchronize(cb_context* ctx) {
  CB_CHECK(ctx, CB_ERR_INVALID, "ctx is null");
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  return CB_OK;
}

int cb_context_device_info(cb_context* ctx, int* sm_count, size_t* hbm_bytes, char* name64) {
  CB_CHECK(ctx, CB_ERR_INVALID, "ctx is null");
  if (sm_count) *sm_count = ctx->sm_count;
  if (hbm_bytes) *hbm_bytes = ctx->hbm_bytes;
  if (name64) snprintf(name64, 64, "%s", ctx->name);
  return CB_OK;
}

uint64_t cb_context_kernel_launches(cb_context* ctx) { return ctx ? ctx->launches : 0; }

int cb_context_flush_l2(cb_context* ctx) {
  CB_CHECK(ctx, CB_ERR_INVALID, "ctx is null");
  CB_CUDA(cudaSetDevice(ctx->device));
  if (!ctx->d_flush) {
    ctx->flush_bytes = std::max<size_t>((size_t)256 << 20, 2 * ctx->l2_bytes);
    // not from ctx->mem: taken from the pool, this buffer would claim memory that the calls timed after a flush
    // then have to map again
    CB_CUDA(cudaMalloc(&ctx->d_flush, ctx->flush_bytes));
  }
  CB_CUDA(cudaMemsetAsync(ctx->d_flush, 0x5a, ctx->flush_bytes, ctx->stream));
  return CB_OK;
}

int cb_comm_unique_id(void* out_128_bytes) { return nccl_unique_id(out_128_bytes); }

int cb_context_init_comm(cb_context* ctx, const void* id, int rank, int world) {
  CB_CHECK(ctx && id, CB_ERR_INVALID, "null argument");
  CB_CHECK(world >= 1 && rank >= 0 && rank < world, CB_ERR_INVALID, "bad rank/world");
  CB_CUDA(cudaSetDevice(ctx->device));
  CB_CHECK(world <= kMaxRanks, CB_ERR_UNSUPPORTED, "at most 16 ranks per communicator");
  CB_TRY(nccl_init(ctx, id, rank, world));
  // until cb_comm_ipc_attach() maps the peers' exchange tables, reductions go through NCCL
  ctx->ex_ready = (world == 1);
  return CB_OK;
}

int cb_comm_ipc_handle(cb_context* ctx, void* out_64_bytes) {
  CB_CHECK(ctx && out_64_bytes, CB_ERR_INVALID, "null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  CB_CUDA(cudaSetDevice(ctx->device));
  cudaIpcMemHandle_t h;
  CB_CUDA(cudaIpcGetMemHandle(&h, ctx->d_xchg));
  std::memcpy(out_64_bytes, &h, sizeof(h));
  return CB_OK;
}

int cb_comm_ipc_attach(cb_context* ctx, const void* handles) {
  CB_CHECK(ctx && handles, CB_ERR_INVALID, "null argument");
  CB_CHECK(ctx->world >= 1 && ctx->world <= kMaxRanks, CB_ERR_INVALID, "call cb_context_init_comm first");
  CB_CUDA(cudaSetDevice(ctx->device));
  // One attach per context: the exchange tables keep the flag values of earlier passes, so a second mapping (with
  // the pass counter restarted) could be satisfied by stale flags. A new communicator needs a new context.
  CB_CHECK(!ctx->ex_attached, CB_ERR_INVALID, "cb_comm_ipc_attach was already called on this context");
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  for (int p = 0; p < ctx->world; ++p) {
    if (p == ctx->rank) {
      ctx->peer_xchg[p] = ctx->d_xchg;
      continue;
    }
    cudaIpcMemHandle_t h;
    std::memcpy(&h, reinterpret_cast<const char*>(handles) + 64 * (size_t)p, sizeof(h));
    void* ptr = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      set_error("cudaIpcOpenMemHandle(rank %d) failed: %s (fused exchange unavailable, NCCL path stays active)", p,
                cudaGetErrorString(e));
      (void)cudaGetLastError();
      return CB_ERR_CUDA;
    }
    ctx->peer_xchg[p] = ptr;
  }
  // The tables were zeroed when the context was created and are only ever written by passes with
  // world > 1, so they are still zero here; do NOT clear them now — a faster peer may already be
  // writing its first row. The launcher barriers after this call before the first pass anyway.
  ctx->seq = 0;
  ctx->h_sync[0] = 0;
  CB_TRY(upload_peer_tables(ctx));
  ctx->ex_ready = true;
  ctx->ex_attached = true;
  return CB_OK;
}

int cb_comm_ipc_detach(cb_context* ctx) {
  CB_CHECK(ctx, CB_ERR_INVALID, "ctx is null");
  if (ctx->world > 1) ctx->ex_ready = false;  // every later pass reduces through NCCL; the mappings stay harmlessly open
  return CB_OK;
}

int cb_context_comm_info(cb_context* ctx, int* rank, int* world) {
  CB_CHECK(ctx, CB_ERR_INVALID, "ctx is null");
  if (rank) *rank = ctx->rank;
  if (world) *world = ctx->world;
  return CB_OK;
}

// ---- clouds -------------------------------------------------------------------------------------
// d_raw (and d_raw_nrm) of a new cloud, from its scope
static int alloc_raw(cb_cloud* c, bool normals) {
  if (c->n == 0) return CB_OK;
  CB_TRY(c->mem.alloc(&c->d_raw, 3 * c->n));
  if (normals) CB_TRY(c->mem.alloc(&c->d_raw_nrm, 3 * c->n));
  return CB_OK;
}

static int upload_raw(cb_cloud* c, const float* xyz, const float* nrm, cudaMemcpyKind kind, cudaStream_t s) {
  if (c->n == 0) return CB_OK;
  CB_CUDA(cudaMemcpyAsync(c->d_raw, xyz, 3 * c->n * sizeof(float), kind, s));
  if (nrm) CB_CUDA(cudaMemcpyAsync(c->d_raw_nrm, nrm, 3 * c->n * sizeof(float), kind, s));
  return CB_OK;
}

static int cloud_fill(cb_cloud* c, const float* xyz, const float* normals, cudaMemcpyKind kind) {
  CB_TRY(alloc_raw(c, normals));
  CB_TRY(upload_raw(c, xyz, normals, kind, c->ctx->stream));
  // the caller's buffers may be released as soon as this returns
  if (c->n > 0) CB_CUDA(cudaStreamSynchronize(c->ctx->stream));
  return CB_OK;
}

static int cloud_create_common(cb_context* ctx, const float* xyz, const float* normals, size_t n, uint64_t off,
                               cudaMemcpyKind kind, cb_cloud** out) {
  CB_CHECK(ctx && out, CB_ERR_INVALID, "null argument");
  CB_CHECK(n == 0 || xyz, CB_ERR_INVALID, "xyz is null");
  CB_CHECK(n < (1ull << 31), CB_ERR_INVALID, "point sets of >= 2^31 points are not supported");
  CB_CUDA(cudaSetDevice(ctx->device));
  cb_cloud* c = new cb_cloud(ctx, n, off);
  const int rc = cloud_fill(c, xyz, normals, kind);
  if (rc != CB_OK) {
    delete c;
    return rc;
  }
  *out = c;
  return CB_OK;
}

static int pair_fill(cb_cloud* a, const float* xyz_a, const float* normals_a, cb_cloud* b, const float* xyz_b,
                     const float* normals_b) {
  cb_context* ctx = a->ctx;
  ScopedEvents ev;
  CB_TRY(ev.create());
  // allocations are stream-ordered on the main stream; the copy stream starts after them
  CB_TRY(alloc_raw(a, normals_a));
  CB_TRY(alloc_raw(b, normals_b));
  CB_CUDA(cudaEventRecord(ev.e0, ctx->stream));
  CB_CUDA(cudaStreamWaitEvent(ctx->copy_stream, ev.e0, 0));
  CB_TRY(upload_raw(a, xyz_a, normals_a, cudaMemcpyHostToDevice, ctx->stream));
  CB_TRY(upload_raw(b, xyz_b, normals_b, cudaMemcpyHostToDevice, ctx->copy_stream));
  CB_CUDA(cudaEventRecord(ev.e1, ctx->copy_stream));
  CB_TRY(ensure_index(a));  // host-blocking in places; the second upload proceeds meanwhile
  CB_CUDA(cudaStreamWaitEvent(ctx->stream, ev.e1, 0));
  CB_TRY(ensure_index(b));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  return CB_OK;
}

// Two clouds at once (the constructor arguments of an ICP object): the host-to-device copy of the second runs on
// a second stream while the grid index of the first is built, so its PCIe time disappears from the critical path
// when the caller's buffers are pinned (pageable buffers make the copy synchronous: same result, no overlap).
// Both clouds are indexed when the call returns and the caller's buffers may be released.
int cb_cloud_create_pair(cb_context* ctx, const float* xyz_a, const float* normals_a, size_t n_a, uint64_t offset_a,
                         const float* xyz_b, const float* normals_b, size_t n_b, uint64_t offset_b, cb_cloud** out_a,
                         cb_cloud** out_b) {
  CB_CHECK(ctx && out_a && out_b, CB_ERR_INVALID, "null argument");
  CB_CHECK((n_a == 0 || xyz_a) && (n_b == 0 || xyz_b), CB_ERR_INVALID, "xyz is null");
  CB_CHECK(n_a < (1ull << 31) && n_b < (1ull << 31), CB_ERR_INVALID, "point sets of >= 2^31 points are not supported");
  CB_CUDA(cudaSetDevice(ctx->device));
  *out_a = *out_b = nullptr;
  if (!ctx->copy_stream) CB_CUDA(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
  cb_cloud* a = new cb_cloud(ctx, n_a, offset_a);
  cb_cloud* b = new cb_cloud(ctx, n_b, offset_b);
  const int rc = pair_fill(a, xyz_a, normals_a, b, xyz_b, normals_b);
  if (rc != CB_OK) {  // the failing call has set the message
    cudaStreamSynchronize(ctx->copy_stream);  // b's upload may still be writing into its buffers
    delete a;
    delete b;
    return rc;
  }
  *out_a = a;
  *out_b = b;
  return CB_OK;
}

// Fills a new cloud from one rank's block of points [first, first + n_block) (host or device memory, `kind`): each
// rank copies only its block into the zero-initialised arrays, and with several ranks one integer-sum all-reduce of
// them is an exact all-gather of bit patterns. Collective when ctx->world > 1.
static int fill_replicated(cb_cloud* c, const float* xyz_block, const float* normals_block, size_t n_block,
                           uint64_t first, cudaMemcpyKind kind) {
  cb_context* ctx = c->ctx;
  const size_t words = 3 * c->n;
  if (words == 0) return CB_OK;
  for (int pass = 0; pass < (normals_block ? 2 : 1); ++pass) {
    float** d = pass == 0 ? &c->d_raw : &c->d_raw_nrm;
    CB_TRY(c->mem.alloc(d, words));
    if (ctx->world > 1) CB_CUDA(cudaMemsetAsync(*d, 0, words * sizeof(float), ctx->stream));
    if (n_block)
      CB_CUDA(cudaMemcpyAsync(*d + 3 * first, pass == 0 ? xyz_block : normals_block, 3 * n_block * sizeof(float), kind,
                              ctx->stream));
    if (ctx->world > 1) CB_TRY(nccl_allreduce_sum_u32(ctx, reinterpret_cast<uint32_t*>(*d), words));
  }
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  return CB_OK;
}

// A cloud every rank needs in full (the destination cloud of a sharded ICP), created from its contiguous blocks: each
// rank uploads ONLY its block over its own PCIe link, the blocks are exchanged over NVLink (fill_replicated). Replaces
// N uploads of the whole cloud (N x the PCIe time for the same bytes) when the caller's data is already partitioned - or
// cheaply sliceable, as in bench.py's end-to-end leg. Collective: every rank of the communicator calls it with the same
// n_total and the same presence of normals (a rank with an empty block passes any non-null pointer).
int cb_cloud_create_replicated(cb_context* ctx, const float* xyz_block, const float* normals_block, size_t n_block,
                               uint64_t first_index, size_t n_total, cb_cloud** out) {
  CB_CHECK(ctx && out, CB_ERR_INVALID, "null argument");
  CB_CHECK(n_block == 0 || xyz_block, CB_ERR_INVALID, "xyz is null");
  CB_CHECK(first_index + n_block <= n_total, CB_ERR_INVALID, "block outside the cloud");
  CB_CHECK(n_total < (1ull << 31), CB_ERR_INVALID, "point sets of >= 2^31 points are not supported");
  CB_CUDA(cudaSetDevice(ctx->device));
  *out = nullptr;
  cb_cloud* c = new cb_cloud(ctx, n_total, 0);
  const int rc = fill_replicated(c, xyz_block, normals_block, n_block, first_index, cudaMemcpyHostToDevice);
  if (rc != CB_OK) {
    delete c;
    return rc;
  }
  *out = c;
  return CB_OK;
}

int cb_cloud_create(cb_context* ctx, const float* xyz, const float* normals, size_t n, uint64_t index_offset,
                    cb_cloud** out) {
  return cloud_create_common(ctx, xyz, normals, n, index_offset, cudaMemcpyHostToDevice, out);
}

int cb_cloud_create_from_device(cb_context* ctx, const float* d_xyz, const float* d_normals, size_t n,
                                uint64_t index_offset, cb_cloud** out) {
  return cloud_create_common(ctx, d_xyz, d_normals, n, index_offset, cudaMemcpyDeviceToDevice, out);
}

void cb_cloud_destroy(cb_cloud* c) {
  if (!c) return;
  cudaSetDevice(c->ctx->device);
  cudaStreamSynchronize(c->ctx->stream);
  delete c;
}

size_t cb_cloud_size(const cb_cloud* c) { return c ? c->n : 0; }

// ---- D-dimensional vector sets --------------------------------------------------------------------
static int vectors_create_common(cb_context* ctx, const float* data, size_t n, int D, cudaMemcpyKind kind,
                                 cb_vectors** out) {
  CB_CHECK(ctx && out, CB_ERR_INVALID, "null argument");
  CB_CHECK(n == 0 || data, CB_ERR_INVALID, "data is null");
  CB_CHECK(D > 0, CB_ERR_INVALID, "D must be >= 1");
  CB_CHECK(n < (1ull << 31), CB_ERR_INVALID, "vector sets of >= 2^31 rows are not supported");
  CB_CUDA(cudaSetDevice(ctx->device));
  *out = nullptr;
  cb_vectors* v = new cb_vectors(ctx, n, D);
  auto fill = [&]() -> int {
    CB_TRY(v->mem.alloc(&v->d_raw, n * (size_t)D));
    if (n) CB_CUDA(cudaMemcpyAsync(v->d_raw, data, n * (size_t)D * sizeof(float), kind, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    return CB_OK;
  };
  const int rc = fill();
  if (rc != CB_OK) {
    delete v;
    return rc;
  }
  *out = v;
  return CB_OK;
}

int cb_vectors_create(cb_context* ctx, const float* data, size_t n, int D, cb_vectors** out) {
  return vectors_create_common(ctx, data, n, D, cudaMemcpyHostToDevice, out);
}

int cb_vectors_create_from_device(cb_context* ctx, const float* d_data, size_t n, int D, cb_vectors** out) {
  return vectors_create_common(ctx, d_data, n, D, cudaMemcpyDeviceToDevice, out);
}

void cb_vectors_destroy(cb_vectors* v) {
  if (!v) return;
  cudaSetDevice(v->ctx->device);
  cudaStreamSynchronize(v->ctx->stream);
  delete v;
}

size_t cb_vectors_size(const cb_vectors* v) { return v ? v->n : 0; }

int cb_cloud_grid_info(const cb_cloud* c, float* cell_edge, int* dims3, double* mean_occupancy) {
  CB_CHECK(c, CB_ERR_INVALID, "cloud is null");
  CB_TRY(ensure_index(const_cast<cb_cloud*>(c)));
  if (cell_edge) *cell_edge = 1.0f / c->inv_h;
  if (dims3) {
    dims3[0] = c->nx;
    dims3[1] = c->ny;
    dims3[2] = c->nz;
  }
  if (mean_occupancy) *mean_occupancy = c->mean_occ;
  return CB_OK;
}

// ---- nearest neighbour ----------------------------------------------------------------------------
static int knn1_device(cb_context* ctx, const cb_cloud* ref, const cb_cloud* qry, const float* T12, float max_d2,
                       DeviceScope& scope, int** d_idx_out, float** d_d2_out) {
  CB_CHECK(ctx && ref && qry, CB_ERR_INVALID, "null argument");
  CB_CHECK(ref->ctx == ctx && qry->ctx == ctx, CB_ERR_INVALID, "cloud belongs to another context");
  CB_CUDA(cudaSetDevice(ctx->device));
  CB_TRY(ensure_index(const_cast<cb_cloud*>(ref)));
  CB_TRY(ensure_index(const_cast<cb_cloud*>(qry)));
  int* d_idx = nullptr;
  float* d_d2 = nullptr;
  CB_TRY(scope.alloc(&d_idx, qry->n));
  CB_TRY(scope.alloc(&d_d2, qry->n));
  IcpArgs a{};
  a.dst = grid_view(ref);
  a.src_pts = qry->d_pts;
  a.src_nrm = nullptr;
  a.n_src = (uint32_t)qry->n;
  a.T = to_rigid(T12);
  a.Tin = to_rigid(nullptr);
  a.max_d2 = max_d2;
  a.out_idx = d_idx;
  a.out_d2 = d_d2;
  CB_TRY(launch_icp_pass(ctx, a, kModeKnn, true, false, false));
  *d_idx_out = d_idx;
  *d_d2_out = d_d2;
  return CB_OK;
}

int cb_knn1_radius(cb_context* ctx, const cb_cloud* ref, const cb_cloud* qry, const float* T12, float max_d2,
                   int64_t* idx, float* d2) {
  DeviceScope scope(ctx);
  int* d_idx = nullptr;
  float* d_d2 = nullptr;
  CB_TRY(knn1_device(ctx, ref, qry, T12, max_d2, scope, &d_idx, &d_d2));
  const size_t nq = qry->n;
  std::vector<int> h_idx(nq);
  if (nq) {
    CB_CUDA(cudaMemcpyAsync(h_idx.data(), d_idx, nq * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    if (d2) CB_CUDA(cudaMemcpyAsync(d2, d_d2, nq * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  }
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  if (idx)
    for (size_t i = 0; i < nq; i++) idx[i] = h_idx[i] < 0 ? -1 : (int64_t)h_idx[i] + (int64_t)ref->index_offset;
  return CB_OK;
}

int cb_find_correspondences(cb_context* ctx, const cb_cloud* ref, const cb_cloud* qry, const float* T12,
                            float max_d2, uint64_t* index_first, uint64_t* index_second, float* value,
                            size_t* count) {
  CB_CHECK(count, CB_ERR_INVALID, "count is null");
  *count = 0;
  if (ref && ref->n == 0) return CB_OK;  // correspondence_search_kd_tree_utilities.hpp:16-19
  DeviceScope scope(ctx);
  int* d_idx = nullptr;
  float* d_d2 = nullptr;
  CB_TRY(knn1_device(ctx, ref, qry, T12, max_d2, scope, &d_idx, &d_d2));
  const size_t nq = qry->n;
  std::vector<int> h_idx(nq);
  std::vector<float> h_d2(nq);
  if (nq) {
    CB_CUDA(cudaMemcpyAsync(h_idx.data(), d_idx, nq * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaMemcpyAsync(h_d2.data(), d_d2, nq * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  }
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  size_t k = 0;  // compaction in query order (:45-50)
  for (size_t i = 0; i < nq; i++) {
    if (h_idx[i] < 0) continue;
    if (index_first) index_first[k] = (uint64_t)h_idx[i] + ref->index_offset;
    if (index_second) index_second[k] = (uint64_t)i + qry->index_offset;
    if (value) value[k] = h_d2[i];
    ++k;
  }
  *count = k;
  return CB_OK;
}

int cb_transform_points(cb_context* ctx, const float* T12, const float* xyz, size_t n, float* out) {
  CB_CHECK(ctx && T12 && (n == 0 || (xyz && out)), CB_ERR_INVALID, "null argument");
  if (n == 0) return CB_OK;
  CB_CUDA(cudaSetDevice(ctx->device));
  DeviceScope scope(ctx);
  float *d_in = nullptr, *d_out = nullptr;
  CB_TRY(scope.alloc(&d_in, 3 * n));
  CB_TRY(scope.alloc(&d_out, 3 * n));
  CB_CUDA(cudaMemcpyAsync(d_in, xyz, 3 * n * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  CB_TRY(launch_transform_points(ctx, to_rigid(T12), d_in, n, d_out));
  CB_CUDA(cudaMemcpyAsync(out, d_out, 3 * n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  return CB_OK;
}

// ---- ICP ------------------------------------------------------------------------------------------
void cb_icp_default_params(cb_icp_params* p) {
  if (!p) return;
  std::memset(p, 0, sizeof(*p));
  p->metric = CB_ICP_POINT_TO_POINT;
  p->max_iter = 15;                  // icp_base.hpp:24
  p->tol = 1e-5f;                    // icp_base.hpp:25
  p->max_d2 = (float)(0.01 * 0.01);  // correspondence_search_kd_tree.hpp:49
  p->w_pt = 0.f;                     // icp_single_transform_combined_metric.hpp:46
  p->w_pl = 1.f;                     // :47
  p->max_opt_iter = 1;               // :44
  p->opt_tol = 1e-5f;                // :45
  t34_identity(p->T_init);
  p->search_dir = CB_SECOND_TO_FIRST;  // correspondence_search_kd_tree.hpp:46-50
  p->inlier_fraction = 1.0;
}

// mean of the finite points of a cloud over all ranks (rowwise().mean(), icp_single_transform_combined_metric.hpp:51-58,
// on the cloud without its NaN / Inf points): the pivots of every ICP metric. The searches never match a non-finite
// point, so skipping them keeps the pivots, and with them the transform, finite (DESIGN §6).
static int global_mean(cb_context* ctx, const cb_cloud* c, bool allreduce, float* mean3) {
  const float zero[3] = {0, 0, 0};
  CB_TRY(launch_moments(ctx, c->d_raw, c->n, zero, /*finite_only=*/true));
  double m[kMomentValues];
  CB_TRY(fetch_result(ctx, kMomentValues, allreduce, m));
  for (int r = 0; r < 3; r++) mean3[r] = (m[0] > 0) ? (float)(m[1 + r] / m[0]) : 0.f;
  return CB_OK;
}

static int icp_init(cb_icp* icp) {
  // dst is replicated on every rank, src is sharded: only the src mean needs the all-reduce
  CB_TRY(global_mean(icp->ctx, icp->dst, false, icp->dst_mean));
  CB_TRY(global_mean(icp->ctx, icp->src, true, icp->src_mean));
  CB_TRY(icp->mem.alloc(&icp->d_nn_pos, icp->src->n));
  CB_TRY(icp->mem.alloc(&icp->d_nn_d2, icp->src->n));
  return CB_OK;
}

int cb_icp_create(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src, cb_icp** out) {
  CB_CHECK(ctx && dst && src && out, CB_ERR_INVALID, "null argument");
  CB_CHECK(dst->ctx == ctx && src->ctx == ctx, CB_ERR_INVALID, "cloud belongs to another context");
  CB_CUDA(cudaSetDevice(ctx->device));
  CB_TRY(ensure_index(const_cast<cb_cloud*>(dst)));
  CB_TRY(ensure_index(const_cast<cb_cloud*>(src)));
  cb_icp* icp = new cb_icp(ctx, dst, src);
  const int rc = icp_init(icp);
  if (rc != CB_OK) {
    delete icp;
    return rc;
  }
  *out = icp;
  return CB_OK;
}

void cb_icp_destroy(cb_icp* icp) {
  if (!icp) return;
  cudaSetDevice(icp->ctx->device);
  cudaStreamSynchronize(icp->ctx->stream);
  delete icp->src_full;
  for (cudaEvent_t e : icp->batch_ev)
    if (e) cudaEventDestroy(e);
  for (cudaEvent_t e : icp->events) cudaEventDestroy(e);
  delete icp;
}

static int icp_fill_args(cb_icp* icp, const cb_icp_params* prm, const float* T, const float* Tin, bool store,
                         IcpArgs* a) {
  std::memset(a, 0, sizeof(*a));
  a->dst = grid_view(icp->dst);
  a->src_pts = icp->src->d_pts;
  a->src_nrm = (prm->metric == CB_ICP_COMBINED) ? icp->src->d_nrm : nullptr;
  a->n_src = (uint32_t)icp->src->n;
  a->T = to_rigid(T);
  a->Tin = to_rigid(Tin);
  a->max_d2 = prm->max_d2;
  a->w_pt = prm->w_pt;
  a->w_pl = prm->w_pl;
  a->wk_pt = prm->pt_weight_kind == CB_WEIGHT_RBF;
  a->wk_pl = prm->pl_weight_kind == CB_WEIGHT_RBF;
  a->wc_pt = prm->pt_weight_coeff;
  a->wc_pl = prm->pl_weight_coeff;
  for (int r = 0; r < 3; r++) a->dm[r] = icp->dst_mean[r];
  float smt[3];
  apply_point(T, icp->src_mean, smt);  // this->transform_ * src_mean_  (:189/:196)
  for (int r = 0; r < 3; r++) a->sm[r] = smt[r];
  // The per-query result is only written when something will read it back (inner Gauss-Newton
  // iterations >= 2, cb_icp_accumulate); cb_icp_correspondences re-runs the search otherwise.
  // The match positions are always kept: they seed the next iteration's search (warm start, warp_search.cuh).
  a->warm_pos = icp->warm_ok ? icp->d_nn_pos : nullptr;
  a->nn_pos = icp->d_nn_pos;
  a->nn_d2 = store ? icp->d_nn_d2 : nullptr;
  std::memcpy(icp->T_search, T, sizeof(icp->T_search));
  icp->max_d2_search = prm->max_d2;
  icp->nn_stored = store;
  return CB_OK;
}

// Totals of the last reduction pass: through the fused exchange when the pass carried it (no stream
// synchronisation: the host polls its mailbox), else all-reduce (NCCL) + copy + synchronise.
static int icp_fetch(cb_context* ctx, int count, double* out, bool allreduce = true) {
  if (ctx->pass_armed) return wait_exchange(ctx, count, out);
  return fetch_result(ctx, count, allreduce, out);
}

// Non-default correspondence-engine modes with several ranks. Their filters rank ALL pairs globally (closest
// fraction, closest pair per destination point) and FIRST_TO_SECOND searches among ALL transformed source points, so a
// shard cannot decide anything alone. Every rank therefore holds the whole source cloud (its blocks all-gathered once
// over NVLink: exact integer-sum all-reduce, as cb_cloud_create_replicated) and runs the same single-GPU list pipeline
// on it: identical lists, sums and transforms on every rank, no all-reduce per iteration - correct and rank-consistent,
// not faster than one GPU. The shards must have been created with index_offset = their first global index.
static int ensure_src_full(cb_icp* icp) {
  cb_context* ctx = icp->ctx;
  if (ctx->world <= 1 || icp->src_full) return CB_OK;
  const cb_cloud* src = icp->src;
  // total size and normals presence over all ranks
  double h[2] = {(double)src->n, src->d_raw_nrm ? 1.0 : 0.0};
  CB_CUDA(cudaMemcpyAsync(ctx->d_result, h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream));
  double tot[2];
  CB_TRY(fetch_result(ctx, 2, true, tot));
  const size_t n_total = (size_t)(tot[0] + 0.5);
  CB_CHECK(src->index_offset + src->n <= n_total, CB_ERR_INVALID,
           "engine modes across ranks: the source shards need index_offset = their first global index");
  const bool nrm = tot[1] > 0.5;
  CB_CHECK(!nrm || (int)(tot[1] + 0.5) == ctx->world, CB_ERR_INVALID, "source normals on some ranks only");
  // (nrm: every rank has normals; otherwise none has)
  cb_cloud* c = new cb_cloud(ctx, n_total, 0);
  int rc = fill_replicated(c, src->d_raw, src->d_raw_nrm, src->n, src->index_offset, cudaMemcpyDeviceToDevice);
  if (rc == CB_OK) rc = ensure_index(c);
  if (rc != CB_OK) {
    delete c;
    return rc;
  }
  icp->src_full = c;
  return CB_OK;
}

// the source cloud the engine modes work on: the whole cloud (replicated) with several ranks, else the caller's
static const cb_cloud* esrc(const cb_icp* icp) { return (icp->ctx->world > 1 && icp->src_full) ? icp->src_full : icp->src; }

// the correspondence list path (icp_engine.cu): non-default engine options, or features attached
static bool icp_engine(const cb_icp* icp, const cb_icp_params* prm) {
  return engine_mode(prm) || icp->feat.kind != CB_FEATURES_POINT;
}

// With a projection attached (cb_icp_set_projection) the kd-tree-only options have no meaning.
static int check_projective(const cb_icp* icp, const cb_icp_params* prm) {
  if (!icp->proj.on) return CB_OK;
  CB_CHECK(prm->search_dir == CB_SECOND_TO_FIRST && !prm->require_reciprocal && !prm->one_to_one &&
               icp->feat.kind == CB_FEATURES_POINT,
           CB_ERR_INVALID, "projective search: search_dir, require_reciprocal, one_to_one and features are kd-tree options");
  return CB_OK;
}

// The projective search's per-query result under a->T into a->nn_pos / a->nn_d2 (filled with store = true), for the
// passes that accumulate without a search.
static int projective_pass_input(cb_icp* icp, const IcpArgs& a) {
  return launch_projective_search(icp->ctx, icp->proj, icp->src->d_pts, (uint32_t)icp->src->n, icp->dst->d_pts, a.T,
                                  a.max_d2, a.nn_pos, a.nn_d2, nullptr, nullptr);
}

// One estimator call of updateEstimate(): returns tform_iter (already un-centred), and the
// correspondence count of the search pass. k0/k1 (nullable) are recorded around the search kernel.

static int icp_update(cb_icp* icp, const cb_icp_params* prm, const float* T, float* Titer, double* n_corr,
                      cudaEvent_t k0, cudaEvent_t k1) {
  cb_context* ctx = icp->ctx;
  IcpArgs a;
  double sums[kMaxValues];
  const bool engine = icp_engine(icp, prm);
  icp->engine_last = engine;
  if (engine) {
    // updateCorrespondences(): the explicit list (icp_engine.cu); the passes below accumulate over it
    if (k0) CB_CUDA(cudaEventRecord(k0, ctx->stream));
    CB_TRY(ensure_src_full(icp));
    CB_TRY(engine_find_pairs(ctx, icp->mem, icp->dst, esrc(icp), prm, T, &icp->pairs, &icp->feat, &icp->proj));
    if (k1) CB_CUDA(cudaEventRecord(k1, ctx->stream));
  }
  const bool proj = icp->proj.on && !engine;
  if (prm->metric == CB_ICP_POINT_TO_POINT) {
    CB_TRY(icp_fill_args(icp, prm, T, nullptr, proj, &a));
    if (engine) {
      // moments about the pivots (dst mean, T * src mean): no cancellation for clouds far from the origin
      CB_TRY(launch_pairs_pass(ctx, a, icp->pairs, icp->dst, esrc(icp), kModeP2PCentered, false, false));
      CB_TRY(icp_fetch(ctx, kP2PValues, sums, /*allreduce=*/false));  // every rank accumulated the whole list
      kabsch_from_pivoted_moments(sums, a.dm, a.sm, Titer);
      *n_corr = sums[0];
      icp->nn_valid = true;
      icp->nn_stored = false;
      return CB_OK;
    }
    if (k0) CB_CUDA(cudaEventRecord(k0, ctx->stream));
    if (proj) CB_TRY(projective_pass_input(icp, a));
    CB_TRY(launch_icp_pass(ctx, a, kModeP2PCentered, !proj, false, false));
    if (k1) CB_CUDA(cudaEventRecord(k1, ctx->stream));
    CB_TRY(icp_fetch(ctx, kP2PValues, sums));
    kabsch_from_pivoted_moments(sums, a.dm, a.sm, Titer);
    *n_corr = sums[0];
    icp->nn_valid = true;
    icp->warm_ok = true;
    return CB_OK;
  }
  // combined / symmetric Gauss-Newton (transform_estimation.hpp:238-367 / :608-739)
  const bool w_pt_on = prm->w_pt > 0.f, w_pl_on = prm->w_pl > 0.f;
  float Tin[12];
  t34_identity(Tin);
  t34_identity(Titer);
  const bool dst_has_normals = icp->dst->d_nrm != nullptr;
  // has_point_to_plane_terms && dst_p.cols() != dst_n.cols() -> return false with identity (:269-272)
  const bool bail_no_normals = w_pl_on && !dst_has_normals;
  const int max_opt = std::max(prm->max_opt_iter, 0);
  for (int it = 0; it < std::max(max_opt, 1); ++it) {
    // (stores d2 too: the RBF weights of inner passes read it; the projective search writes its result there)
    CB_TRY(icp_fill_args(icp, prm, T, Tin, (max_opt > 1 || proj) && !engine, &a));
    const bool search = (it == 0);
    if (engine) {
      CB_TRY(launch_pairs_pass(ctx, a, icp->pairs, icp->dst, esrc(icp), kModeCombined, w_pt_on,
                               w_pl_on && dst_has_normals));
    } else {
      // the first pass always runs (it is also the correspondence search of this ICP iteration)
      if (search && k0) CB_CUDA(cudaEventRecord(k0, ctx->stream));
      if (search && proj) CB_TRY(projective_pass_input(icp, a));
      CB_TRY(launch_icp_pass(ctx, a, kModeCombined, search && !proj, w_pt_on, w_pl_on && dst_has_normals));
      if (search && k1) CB_CUDA(cudaEventRecord(k1, ctx->stream));
    }
    CB_TRY(icp_fetch(ctx, kCombinedValues, sums, /*allreduce=*/!(engine && ctx->world > 1)));
    if (search) {
      *n_corr = sums[0];
      icp->nn_valid = true;
      icp->warm_ok = !engine;
    }
    const bool has_terms = sums[0] > 0.0 && (w_pt_on || w_pl_on);
    if (!has_terms || bail_no_normals) {
      t34_identity(Titer);
      return CB_OK;
    }
    if (max_opt == 0) break;  // max_iter == 0: loop body never runs, only the un-centring (:365)
    float dn = 0.f;
    float Tnext[12];
    gauss_newton_update(sums, Tin, Tnext, &dn);
    std::memcpy(Tin, Tnext, sizeof(Tin));
    if (dn < prm->opt_tol) break;  // :360-363
  }
  std::memcpy(Titer, Tin, sizeof(Tin));
  float smt[3];
  apply_point(T, icp->src_mean, smt);
  uncenter(Titer, icp->dst_mean, smt);
  return CB_OK;
}

int cb_icp_estimate(cb_icp* icp, const cb_icp_params* prm, cb_icp_result* res) {
  CB_CHECK(icp && prm && res, CB_ERR_INVALID, "null argument");
  CB_CHECK(prm->metric == CB_ICP_POINT_TO_POINT || prm->metric == CB_ICP_COMBINED, CB_ERR_INVALID, "bad metric");
  CB_TRY(check_projective(icp, prm));
  cb_context* ctx = icp->ctx;
  CB_CUDA(cudaSetDevice(ctx->device));
  int hand_over = 0;
  {
    // Default correspondence engine, one Gauss-Newton step per iteration (the reference's defaults): the
    // device-resident loop (icp_loop.cu). prm->host_loop keeps the host-driven loop below; engine modes, inner
    // Gauss-Newton iterations and multi-rank runs without the fused exchange always use it.
    const bool one_step = prm->metric == CB_ICP_POINT_TO_POINT || prm->max_opt_iter == 1;
    if (!prm->host_loop && !icp_engine(icp, prm) && one_step && (ctx->world == 1 || exchange_available(ctx))) {
      const int rc = icp_loop_estimate(icp, prm, res, &hand_over);
      if (rc != CB_OK || !hand_over) return rc;
      // the run is not converging: continue from the device loop's state with the host-driven loop below
    }
  }
  icp->loop_last = false;
  const uint64_t launches0 = ctx->launches;
  const int max_iter = std::max(prm->max_iter, 0);
  // Optional CUDA-event instrumentation, ONE bracket (2 events) per iteration: timing 1 = whole
  // iteration, timing 2 = the search kernel only. Every cudaEventRecord costs the device front end a
  // few microseconds (visible in a %globaltimer trace of the iteration period), so production runs
  // (timing 0) record nothing. Elapsed times are read after the final
  // synchronise: with the fused exchange the host never waits on the stream inside the loop.
  const int timing = prm->timing;
  while (timing != 0 && (int)icp->events.size() < 2 * max_iter) {
    cudaEvent_t e;
    CB_CUDA(cudaEventCreate(&e));
    icp->events.push_back(e);
  }
  float T[12];
  std::memcpy(T, prm->T_init, sizeof(T));  // icp_base.hpp:71
  int iters = 0;
  float last_delta = INFINITY;
  double n_corr = 0;
  icp->nn_valid = false;
  icp->warm_ok = false;
  icp->search_ms = 0;
  const uint64_t loop_launches = hand_over ? res->kernel_launches : 0;
  std::vector<double> loop_iter_ms;
  if (hand_over) {
    // continue the device loop's run: its transform, its iteration count, its matches as warm seeds
    // (d_nn_pos holds sorted dst positions or -1 there too)
    std::memcpy(T, res->T, sizeof(T));
    iters = res->iterations;
    last_delta = res->last_delta;
    n_corr = (double)res->num_corr;
    icp->nn_valid = true;
    icp->warm_ok = true;
    loop_iter_ms = icp->iter_ms;
  }
  const int iters0 = iters;
  while (iters < max_iter) {  // icp_base.hpp:76-84
    if (prm->flush_l2) CB_TRY(cb_context_flush_l2(ctx));
    cudaEvent_t e0 = timing ? icp->events[2 * iters] : nullptr, e1 = timing ? icp->events[2 * iters + 1] : nullptr;
    if (timing == 1) CB_CUDA(cudaEventRecord(e0, ctx->stream));
    float Titer[12];
    // updateCorrespondences() + updateEstimate(): one fused pass (+ stored-correspondence passes
    // for inner Gauss-Newton iterations), reduction (+ exchange), host solve
    CB_TRY(icp_update(icp, prm, T, Titer, &n_corr, timing == 2 ? e0 : nullptr, timing == 2 ? e1 : nullptr));
    reorthonormalize(Titer);           // :207-211
    compose(Titer, T, T);              // :213
    last_delta = update_norm(Titer);   // :214-216
    // recorded AFTER the host solve: the device timestamps it when it gets to it, so the bracket
    // covers kernel + exchange + host solve of this iteration
    if (timing == 1) CB_CUDA(cudaEventRecord(e1, ctx->stream));
    iters++;
    if (last_delta < prm->tol) break;  // icp_base.hpp:83
  }
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  icp->iter_ms.assign(iters, 0.0);
  double total = 0;
  for (int i = 0; i < iters0 && i < (int)loop_iter_ms.size(); i++) {  // the device loop's share of a handed-over run
    icp->iter_ms[i] = loop_iter_ms[i];
    total += loop_iter_ms[i];
    if (timing == 2) icp->search_ms += loop_iter_ms[i];
  }
  for (int i = iters0; i < iters && timing != 0; i++) {
    float ms = 0.f;
    CB_CUDA(cudaEventElapsedTime(&ms, icp->events[2 * i], icp->events[2 * i + 1]));
    if (timing == 1) {
      icp->iter_ms[i] = ms;
      total += ms;
    } else {
      icp->search_ms += ms;
    }
  }
  if (getenv("CB_TRACE_EXCHANGE") && ctx->seq >= 8) {
    // last 6 passes: kernel start -> local reduction -> peers summed -> mailbox flag, and start-to-start period
    unsigned long long prev0 = 0;
    for (unsigned long long q = ctx->seq - 5; q <= ctx->seq; ++q) {
      const unsigned long long* t = ctx->h_sync + 64 + 4 * (q % 64);
      fprintf(stderr, "[rank %d pass %llu] start->reduced %.1f us, reduced->peers %.1f us, peers->flag %.1f us, period %.1f us\n",
              ctx->rank, q, (t[1] - t[0]) * 1e-3, (t[2] - t[1]) * 1e-3, (t[3] - t[2]) * 1e-3,
              prev0 ? (t[0] - prev0) * 1e-3 : 0.0);
      prev0 = t[0];
    }
  }
  std::memcpy(res->T, T, sizeof(T));
  res->iterations = iters;
  res->last_delta = last_delta;
  res->converged = last_delta < prm->tol;
  res->num_corr = (uint64_t)(n_corr + 0.5);
  res->gpu_ms_total = total;
  res->gpu_ms_search = icp->search_ms;
  res->kernel_launches = ctx->launches - launches0 + loop_launches;
  return CB_OK;
}

int cb_icp_iteration_times(cb_icp* icp, double* ms, int cap) {
  CB_CHECK(icp && ms, CB_ERR_INVALID, "null argument");
  const int n = std::min<int>(cap, (int)icp->iter_ms.size());
  for (int i = 0; i < n; i++) ms[i] = icp->iter_ms[i];
  return n;
}

int cb_icp_accumulate(cb_icp* icp, const cb_icp_params* prm, const float* T12, double* sums, int cap) {
  CB_CHECK(icp && prm && T12 && sums, CB_ERR_INVALID, "null argument");
  cb_context* ctx = icp->ctx;
  CB_CUDA(cudaSetDevice(ctx->device));
  CB_TRY(check_projective(icp, prm));
  IcpArgs a;
  double tmp[kMaxValues];
  int nv;
  if (icp->feat.kind != CB_FEATURES_POINT || (icp->proj.on && engine_mode(prm))) {
    // the feature search's or the fraction-filtered projective correspondence list (icp_engine.cu), accumulated like
    // the list path's passes
    const bool p2p = prm->metric == CB_ICP_POINT_TO_POINT;
    nv = p2p ? kP2PValues : kCombinedValues;
    CB_CHECK(p2p || !(prm->w_pl > 0.f) || icp->dst->d_nrm, CB_ERR_INVALID, "dst has no normals");
    CB_CHECK(cap >= nv, CB_ERR_INVALID, "sums buffer too small");
    CB_TRY(engine_find_pairs(ctx, icp->mem, icp->dst, icp->src, prm, T12, &icp->pairs, &icp->feat, &icp->proj));
    CB_TRY(icp_fill_args(icp, prm, T12, nullptr, false, &a));
    CB_TRY(launch_pairs_pass(ctx, a, icp->pairs, icp->dst, icp->src, p2p ? kModeP2P : kModeCombined,
                             !p2p && prm->w_pt > 0.f, !p2p && prm->w_pl > 0.f));
    CB_TRY(icp_fetch(ctx, nv, tmp, /*allreduce=*/false));
    std::memcpy(sums, tmp, nv * sizeof(double));
    icp->engine_last = true;
    icp->nn_valid = true;
    return nv;
  }
  CB_TRY(icp_fill_args(icp, prm, T12, nullptr, true, &a));
  icp->engine_last = false;  // cb_icp_correspondences reads this pass's per-query result
  const bool proj = icp->proj.on;
  if (prm->metric == CB_ICP_POINT_TO_POINT) {
    nv = kP2PValues;
    if (proj) CB_TRY(projective_pass_input(icp, a));
    CB_TRY(launch_icp_pass(ctx, a, kModeP2P, !proj, false, false));
  } else {
    nv = kCombinedValues;
    CB_CHECK(!(prm->w_pl > 0.f) || icp->dst->d_nrm, CB_ERR_INVALID, "dst has no normals");
    if (proj) CB_TRY(projective_pass_input(icp, a));
    CB_TRY(launch_icp_pass(ctx, a, kModeCombined, !proj, prm->w_pt > 0.f, prm->w_pl > 0.f));
  }
  CB_CHECK(cap >= nv, CB_ERR_INVALID, "sums buffer too small");
  CB_TRY(icp_fetch(ctx, nv, tmp));
  std::memcpy(sums, tmp, nv * sizeof(double));
  icp->nn_valid = true;
  return nv;
}

int cb_icp_correspondences(cb_icp* icp, uint64_t* index_first, uint64_t* index_second, float* value, size_t* count) {
  CB_CHECK(icp && count, CB_ERR_INVALID, "null argument");
  CB_CHECK(icp->nn_valid, CB_ERR_INVALID, "no correspondences yet: call cb_icp_estimate first");
  cb_context* ctx = icp->ctx;
  CB_CUDA(cudaSetDevice(ctx->device));
  const size_t ns = icp->src->n;
  *count = 0;
  if (icp->engine_last) {  // the list is already materialised, in the reference's order
    const size_t m = icp->pairs.count;
    if (m == 0) return CB_OK;
    std::vector<uint32_t> f(m), s(m);
    CB_CUDA(cudaMemcpyAsync(f.data(), icp->pairs.first, m * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaMemcpyAsync(s.data(), icp->pairs.second, m * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    if (value) CB_CUDA(cudaMemcpyAsync(value, icp->pairs.d2, m * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    for (size_t k = 0; k < m; k++) {
      if (index_first) index_first[k] = (uint64_t)f[k] + icp->dst->index_offset;
      if (index_second) index_second[k] = (uint64_t)s[k] + esrc(icp)->index_offset;  // (several ranks: the global list)
    }
    *count = m;
    return CB_OK;
  }
  if (ns == 0) return CB_OK;
  if (!icp->nn_stored && icp->proj.on) {  // the device loop's projective run: re-run its last search
    CB_TRY(launch_projective_search(ctx, icp->proj, icp->src->d_pts, (uint32_t)ns, icp->dst->d_pts,
                                    to_rigid(icp->T_search), icp->max_d2_search, icp->d_nn_pos, icp->d_nn_d2, nullptr,
                                    nullptr));
    icp->nn_stored = true;
  }
  if (!icp->nn_stored) {  // re-run the last search, this time keeping the per-query result
    IcpArgs a{};
    a.dst = grid_view(icp->dst);
    a.src_pts = icp->src->d_pts;
    a.n_src = (uint32_t)ns;
    a.T = to_rigid(icp->T_search);
    a.Tin = to_rigid(nullptr);
    a.max_d2 = icp->max_d2_search;
    a.nn_pos = icp->d_nn_pos;
    a.nn_d2 = icp->d_nn_d2;
    CB_TRY(launch_icp_pass(ctx, a, kModeKnn, true, false, false));
    icp->nn_stored = true;
  }
  // nn_pos is indexed by sorted src position and holds sorted dst positions: translate to ORIGINAL indices on the
  // device (one small kernel) and download n_src ints + floats; the compaction in source order stays on the host
  DeviceScope sc(ctx);
  int* d_first = nullptr;
  float* d_val = nullptr;
  CB_TRY(sc.alloc(&d_first, ns));
  CB_TRY(sc.alloc(&d_val, ns));
  CB_TRY(launch_translate_matches(ctx, icp->d_nn_pos, icp->d_nn_d2, icp->src->d_pts, icp->dst->d_pts, (uint32_t)ns, d_first,
                                  d_val));
  std::vector<int> first(ns);
  std::vector<float> val(ns);
  CB_CUDA(cudaMemcpyAsync(first.data(), d_first, ns * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaMemcpyAsync(val.data(), d_val, ns * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  size_t k = 0;
  for (size_t i = 0; i < ns; i++) {
    if (first[i] < 0) continue;
    if (index_first) index_first[k] = (uint64_t)first[i] + icp->dst->index_offset;
    if (index_second) index_second[k] = (uint64_t)i + icp->src->index_offset;
    if (value) value[k] = val[i];
    ++k;
  }
  *count = k;
  return CB_OK;
}

int cb_icp_loop_cache(cb_icp* icp, float* T_search12, int64_t* nearest, uint64_t* searched_last) {
  CB_CHECK(icp, CB_ERR_INVALID, "null argument");
  CB_CHECK(icp->loop_last && icp->h_state, CB_ERR_INVALID, "the last cb_icp_estimate did not run on the device loop");
  cb_context* ctx = icp->ctx;
  CB_CUDA(cudaSetDevice(ctx->device));
  const size_t ns = icp->src->n;
  if (T_search12) std::memcpy(T_search12, icp->T_search, sizeof(icp->T_search));
  if (searched_last) *searched_last = icp->searched_last;
  if (nearest && ns) {
    DeviceScope sc(ctx);
    int* d_first = nullptr;
    CB_TRY(sc.alloc(&d_first, ns));
    CB_TRY(launch_translate_matches(ctx, icp->d_nn_pos, nullptr, icp->src->d_pts, icp->dst->d_pts, (uint32_t)ns, d_first,
                                    nullptr));
    std::vector<int> first(ns);
    CB_CUDA(cudaMemcpyAsync(first.data(), d_first, ns * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CB_CUDA(cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i < ns; i++) nearest[i] = first[i] < 0 ? -1 : (int64_t)first[i] + (int64_t)icp->dst->index_offset;
  }
  return CB_OK;
}

// n x 3 host vectors weighted into one tail slot of an n x tails float4 array (the adaptors' constructors: one fp32
// multiply per component)
static void weight_tails(const float* v, size_t n, float w, int tails, int slot, std::vector<float4>& out) {
  for (size_t i = 0; i < n; i++)
    out[i * tails + slot] = make_float4(rule::mul_rn(w, v[3 * i]), rule::mul_rn(w, v[3 * i + 1]),
                                        rule::mul_rn(w, v[3 * i + 2]), 0.f);
}

int cb_icp_set_features(cb_icp* icp, int kind, const float* dst_normals, const float* dst_colors,
                        const float* src_normals, const float* src_colors, float normal_weight, float color_weight) {
  CB_CHECK(icp, CB_ERR_INVALID, "null argument");
  CB_CHECK(kind >= CB_FEATURES_POINT && kind <= CB_FEATURES_POINT_NORMAL_COLOR, CB_ERR_INVALID, "bad feature kind");
  cb_context* ctx = icp->ctx;
  CB_CHECK(ctx->world == 1, CB_ERR_UNSUPPORTED, "feature search with several ranks");
  const bool nrm = kind == CB_FEATURES_POINT_NORMAL || kind == CB_FEATURES_POINT_NORMAL_COLOR;
  const bool col = kind == CB_FEATURES_POINT_COLOR || kind == CB_FEATURES_POINT_NORMAL_COLOR;
  CB_CHECK(!nrm || (dst_normals && src_normals), CB_ERR_INVALID, "the feature kind needs dst and src normals");
  CB_CHECK(!col || (dst_colors && src_colors), CB_ERR_INVALID, "the feature kind needs dst and src colors");
  CB_CHECK(!nrm || std::isfinite(normal_weight), CB_ERR_INVALID, "normal weight is not finite");
  CB_CHECK(!col || std::isfinite(color_weight), CB_ERR_INVALID, "color weight is not finite");
  CB_CUDA(cudaSetDevice(ctx->device));
  FeatureSet& f = icp->feat;
  for (float4* p : {f.dst_raw, f.dst_sorted, f.src_raw}) CB_TRY(icp->mem.free(p));
  f = FeatureSet();
  icp->nn_valid = false;
  icp->engine_last = false;
  if (kind == CB_FEATURES_POINT) return CB_OK;
  const int tails = rule::feature_tails(kind);
  const size_t nd = icp->dst->n, ns = icp->src->n;
  std::vector<float4> hd(nd * tails), hs(ns * tails);
  int slot = 0;
  if (nrm) {
    weight_tails(dst_normals, nd, normal_weight, tails, slot, hd);
    weight_tails(src_normals, ns, normal_weight, tails, slot, hs);
    ++slot;
  }
  if (col) {
    weight_tails(dst_colors, nd, color_weight, tails, slot, hd);
    weight_tails(src_colors, ns, color_weight, tails, slot, hs);
  }
  FeatureSet nf;
  nf.kind = kind;
  CB_TRY(icp->mem.alloc(&nf.dst_raw, nd * tails));
  CB_TRY(icp->mem.alloc(&nf.dst_sorted, nd * tails));
  CB_TRY(icp->mem.alloc(&nf.src_raw, ns * tails));
  f = nf;  // owned by icp->mem from here on
  CB_CUDA(cudaMemcpyAsync(f.dst_raw, hd.data(), hd.size() * sizeof(float4), cudaMemcpyHostToDevice, ctx->stream));
  CB_CUDA(cudaMemcpyAsync(f.src_raw, hs.data(), hs.size() * sizeof(float4), cudaMemcpyHostToDevice, ctx->stream));
  CB_TRY(launch_feature_gather(ctx, kind, icp->dst->d_pts, (uint32_t)nd, f.dst_raw, nullptr, f.dst_sorted));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));  // the host staging vectors go out of scope
  return CB_OK;
}

int cb_icp_residuals(cb_icp* icp, const cb_icp_params* prm, const float* T12, float* out) {
  CB_CHECK(icp && prm && T12 && out, CB_ERR_INVALID, "null argument");
  cb_context* ctx = icp->ctx;
  CB_CUDA(cudaSetDevice(ctx->device));
  const size_t ns = icp->src->n;
  if (ns == 0) return CB_OK;
  CB_CHECK(prm->metric == CB_ICP_POINT_TO_POINT || icp->dst->d_nrm || icp->dst->n == 0, CB_ERR_INVALID,
           "dst has no normals");
  DeviceScope scope(ctx);
  float* d_out = nullptr;
  CB_TRY(scope.alloc(&d_out, ns));
  CB_TRY(launch_residuals(ctx, grid_view(icp->dst), icp->src->d_pts,
                          prm->metric == CB_ICP_COMBINED ? icp->src->d_nrm : nullptr, (uint32_t)ns, to_rigid(T12),
                          prm->metric, prm->w_pt, prm->w_pl, d_out));
  CB_CUDA(cudaMemcpyAsync(out, d_out, ns * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  return CB_OK;
}

}  // extern "C"
