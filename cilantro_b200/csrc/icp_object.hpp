// The ICP object behind cb_icp_* (product code): shared by the host-driven loop (capi_core.cu) and the
// device-resident loop (icp_loop.cu).
#pragma once
#include "cb_internal.hpp"
#include <vector>

namespace cb {

// State of the device-resident ICP loop (icp_loop.cu): lives in device memory, read by every block at the start of
// an iteration's kernel and rewritten by the ONE thread that finishes the iteration (reduction -> exchange ->
// solve), so consecutive iterations need no host round trip. The host reads it back once per batch of launches.
struct LoopState {
  float T[12];        // current estimate = the transform the NEXT iteration searches with
  float T_prev[12];   // the transform the last executed iteration searched with
  float Titer[12];    // that iteration's update
  float last_delta;   // its norm (icp_single_transform_*_metric.hpp:214-216 / :62-64)
  int iters;          // iterations executed (icp_base.hpp:76-84)
  int done;           // 1 = converged (last_delta < tol), 2 = failed (error): later launches return at once
  int have_prev;      // the per-query cache (match, exclusion radius) is valid relative to T_prev
  int error;          // cb_status of a failed iteration (peer wait timed out)
  int pad_;
  unsigned long long xseq;  // fused-exchange pass number of the last executed iteration (Exchange::seq)
  double n_corr;      // correspondences of the last executed iteration (all ranks)
  unsigned long long searched_cur;   // queries searched so far by the running iteration (this rank)
  unsigned long long searched_last;  // ... by the last executed iteration
  double searched_all;               // the same over ALL ranks (exchanged with the moments: identical everywhere)
  double queries_all;                // source points of all ranks
  double sums[32];    // its reduced moments / normal equations (all ranks)
  // CB_LOOP_TRACE=1: per executed iteration (mod 64): %globaltimer at kernel start / local reduction done /
  // peers' rows summed / state written, the number of queries that needed a search, %globaltimer when the last warp
  // of the grid reached the reduction (its tiles and searches done)
  unsigned long long trace[64][6];
};

}  // namespace cb

struct cb_icp {
  cb_icp(cb_context* c, const cb_cloud* d, const cb_cloud* s) : ctx(c), dst(d), src(s), mem(c) {}
  cb_context* ctx = nullptr;
  const cb_cloud* dst = nullptr;
  const cb_cloud* src = nullptr;
  cb::DeviceScope mem;  // every buffer below (device and pinned host)
  float dst_mean[3] = {0, 0, 0};
  float src_mean[3] = {0, 0, 0};
  int* d_nn_pos = nullptr;  // per sorted src point: sorted dst position of its match, -1 none
  float* d_nn_d2 = nullptr;
  bool nn_valid = false;    // a search has run; T_search / max_d2_search describe it
  bool nn_stored = false;   // d_nn_pos / d_nn_d2 hold that search's per-query result
  bool warm_ok = false;     // d_nn_pos holds the previous iteration's matches of THIS estimate() call
  float T_search[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
  float max_d2_search = 0.f;
  cb::EnginePairs pairs;    // correspondence list of the last iteration in a non-default engine mode
  bool engine_last = false; // the last estimate() went through icp_engine.cu
  cb::FeatureSet feat;      // cb_icp_set_features (tails owned by `mem`)
  double search_ms = 0;  // CUDA-event time of the fused search+accumulate kernels of the last estimate()
  std::vector<cudaEvent_t> events;
  std::vector<double> iter_ms;
  // device-resident loop (icp_loop.cu); the per-query cache lives in d_nn_pos (match) / d_nn_d2 (exclusion radius)
  cb::LoopState* d_state = nullptr;
  cb::LoopState* h_state = nullptr;  // pinned
  cb::LoopState* h_state2 = nullptr; // pinned: the batches' states alternate between the two
  cudaEvent_t batch_ev[2] = {nullptr, nullptr};  // end of a batch + its state copy
  cb_cloud* src_full = nullptr;      // world > 1, engine modes: the whole source cloud replicated on this rank (owned)
  bool loop_last = false;            // the last estimate() ran on the device loop
  uint64_t searched_last = 0;        // queries its last iteration searched again (CB_LOOP_TRACE / cb_icp_loop_cache)
};

namespace cb {
// cb_icp_estimate for the default correspondence engine with one Gauss-Newton step per iteration: all iterations
// enqueued back to back, transform kept on the device (icp_loop.cu).
// *hand_over = 1: the loop stopped after res->iterations iterations because the cache was not paying (the run is not
// converging: a large share of the queries is searched again every iteration); the caller continues from res with the
// host-driven loop, whose plain search is cheaper per searched query.
int icp_loop_estimate(cb_icp* icp, const cb_icp_params* prm, cb_icp_result* res, int* hand_over);
unsigned long long exchange_timeout_ns();
}  // namespace cb
