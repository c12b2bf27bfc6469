// Non-default correspondence-engine modes of the ICP path (product code, sm_90a) — §8(f) rank 3.
// Replaces CorrespondenceSearchKDTree::findCorrespondences(tform) (correspondence_search/
// correspondence_search_kd_tree.hpp:107-229) for search directions FIRST_TO_SECOND / BOTH, reciprocity,
// inlier_fraction < 1 and one_to_one; the default configuration keeps the fused single-kernel path
// (icp_kernels.cu) and never comes here. With feature tails attached (cb_icp_set_features) every configuration comes
// here, and both searches run on the feature distance (feature_search.cu).
//
// Per ICP iteration the correspondence list is materialised on the device in the reference's own order:
//   SECOND_TO_FIRST  q_j = T src_j searched in the dst grid          -> pairs (nn(j), j),   ascending j
//   FIRST_TO_SECOND  dst_i searched in a grid over {T src_j}, which is rebuilt every iteration exactly like
//                    the reference's src_trans_tree_ (:201-203): same transformed coordinates, so indices and
//                    squared distances are bit-identical                -> pairs (i, nn'(i)),  ascending i
//   BOTH             set_union / set_intersection of the two lists on (first, second)
//                    (correspondence_search_kd_tree_utilities.hpp:79-99) -> lexicographic order
//   filterCorrespondencesFraction (core/correspondence.hpp:57-66): ascending value, first llround(f * M)
//   filterCorrespondencesOneToOne (:68-100): per dst (S2F) / src (F2S) point the pair of smallest value,
//                    ascending in that index; BOTH: no-op.
// std::sort leaves the order of equal keys unspecified; here ties are resolved by the position in the list
// the filter received (radix sorts are stable), and the oracle uses the same rule.
// Sorting = radix_sort_pairs_u64 over (key, pair id); accumulation = one thread per pair over the raw
// (original-order) arrays with the same per-pair arithmetic as the fused kernel (icp_accumulate.cuh).
#include "feature_rule.hpp"
#include "feature_search.cuh"
#include "icp_accumulate.cuh"
#include "icp_kernels.cuh"
#include "reduce.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace cb {

namespace {

constexpr int kThreads = 256;

inline int blocks_for(const cb_context* ctx, size_t n) {
  return (int)std::max<size_t>(1, std::min<size_t>((n + kThreads - 1) / kThreads, (size_t)ctx->sm_count * 16));
}

using Dev = DeviceScope;  // scoped stream-ordered allocations (cb_internal.hpp)

// Candidate c of the pre-filter list: c < n_a -> the S2F pair of src point c (when s2f_idx != nullptr),
// else the F2S pair of dst point c - n_a. Validity includes the union / intersection rules of BOTH.
struct Candidates {
  const int* s2f_idx;   // per src point (original order): matched dst index or -1
  const float* s2f_d2;
  const int* f2s_idx;   // per dst point (original order): matched src index or -1
  const float* f2s_d2;
  uint32_t n_a;         // number of S2F candidates (n_src or 0)
  uint32_t n_b;         // number of F2S candidates (n_dst or 0)
  int both;             // direction BOTH
  int reciprocal;
};

__device__ __forceinline__ bool candidate(const Candidates& c, uint32_t k, uint32_t& first, uint32_t& second,
                                          float& d2) {
  if (k < c.n_a) {
    const int i = c.s2f_idx[k];
    if (i < 0) return false;
    if (c.both && c.reciprocal && c.f2s_idx[i] != (int)k) return false;  // set_intersection
    first = (uint32_t)i;
    second = k;
    d2 = c.s2f_d2[k];
    return true;
  }
  const uint32_t i = k - c.n_a;
  const int j = c.f2s_idx[i];
  if (j < 0) return false;
  if (c.both) {
    if (c.reciprocal) return false;                 // the intersection is enumerated from the S2F side
    if (c.s2f_idx[j] == (int)i) return false;       // set_union: the pair is already in the S2F list
  }
  first = i;
  second = (uint32_t)j;
  d2 = c.f2s_d2[i];
  return true;
}

__global__ void candidate_flag_kernel(const Candidates c, uint32_t total, uint32_t* __restrict__ flags) {
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k <= total; k += gridDim.x * blockDim.x) {
    uint32_t f, s;
    float d;
    flags[k] = (k < total && candidate(c, k, f, s, d)) ? 1u : 0u;
  }
}

__global__ void candidate_compact_kernel(const Candidates c, uint32_t total, const uint32_t* __restrict__ scanned,
                                         uint32_t* __restrict__ first, uint32_t* __restrict__ second,
                                         float* __restrict__ d2) {
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < total; k += gridDim.x * blockDim.x) {
    uint32_t f, s;
    float d;
    if (candidate(c, k, f, s, d)) {
      const uint32_t p = scanned[k];
      first[p] = f;
      second[p] = s;
      d2[p] = d;
    }
  }
}

enum KeyKind : int { kKeyLex = 0, kKeyValuePos = 1, kKeyFirstValue = 2, kKeySecondValue = 3 };

// key = (high field << low_bits) | low field, packed tightly so that the radix sort only runs the passes the
// value ranges need (low_bits = width of the low field: index bits, value bits or position bits)
__global__ void pair_key_kernel(const uint32_t* __restrict__ first, const uint32_t* __restrict__ second,
                                const float* __restrict__ d2, uint32_t m, int kind, int low_bits,
                                uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < m; p += gridDim.x * blockDim.x) {
    const uint64_t v = (uint64_t)__float_as_uint(d2[p]);  // d2 >= 0: the bit pattern is monotone
    uint64_t k;
    if (kind == kKeyLex) k = ((uint64_t)first[p] << low_bits) | second[p];
    else if (kind == kKeyValuePos) k = (v << low_bits) | p;
    else if (kind == kKeyFirstValue) k = ((uint64_t)first[p] << low_bits) | v;
    else k = ((uint64_t)second[p] << low_bits) | v;
    keys[p] = k;
    vals[p] = p;
  }
}

__global__ void pair_gather_kernel(const uint32_t* __restrict__ perm, uint32_t m, const uint32_t* __restrict__ f_in,
                                   const uint32_t* __restrict__ s_in, const float* __restrict__ d_in,
                                   uint32_t* __restrict__ f_out, uint32_t* __restrict__ s_out,
                                   float* __restrict__ d_out) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < m; p += gridDim.x * blockDim.x) {
    const uint32_t q = perm[p];
    f_out[p] = f_in[q];
    s_out[p] = s_in[q];
    d_out[p] = d_in[q];
  }
}

// one-to-one: after the stable sort on (index, value) keep the head of every index group
__global__ void group_head_flag_kernel(const uint32_t* __restrict__ index, uint32_t m, uint32_t* __restrict__ flags) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p <= m; p += gridDim.x * blockDim.x)
    flags[p] = (p < m && (p == 0 || index[p] != index[p - 1])) ? 1u : 0u;
}

__global__ void flagged_compact_kernel(const uint32_t* __restrict__ index, uint32_t m,
                                       const uint32_t* __restrict__ scanned, const uint32_t* __restrict__ f_in,
                                       const uint32_t* __restrict__ s_in, const float* __restrict__ d_in,
                                       uint32_t* __restrict__ f_out, uint32_t* __restrict__ s_out,
                                       float* __restrict__ d_out) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < m; p += gridDim.x * blockDim.x) {
    if (p == 0 || index[p] != index[p - 1]) {
      const uint32_t q = scanned[p];
      f_out[q] = f_in[p];
      s_out[q] = s_in[p];
      d_out[q] = d_in[p];
    }
  }
}

struct PairBufs {
  uint32_t *f[2], *s[2];
  float* d[2];
  uint64_t* keys[2];
  uint32_t* vals[2];
  uint32_t* flags;
  int cur = 0;
};

int sort_pairs(cb_context* ctx, PairBufs& b, uint32_t m, int kind, int high_bits, int low_bits) {
  if (m <= 1) return CB_OK;
  const int nb = blocks_for(ctx, m);
  pair_key_kernel<<<nb, kThreads, 0, ctx->stream>>>(b.f[b.cur], b.s[b.cur], b.d[b.cur], m, kind, low_bits, b.keys[0],
                                                   b.vals[0]);
  ctx->launches += 1;
  CB_TRY(radix_sort_pairs_u64(ctx, b.keys[0], b.vals[0], b.keys[1], b.vals[1], m, high_bits + low_bits));
  pair_gather_kernel<<<nb, kThreads, 0, ctx->stream>>>(b.vals[0], m, b.f[b.cur], b.s[b.cur], b.d[b.cur],
                                                      b.f[b.cur ^ 1], b.s[b.cur ^ 1], b.d[b.cur ^ 1]);
  ctx->launches += 1;
  CB_CUDA(cudaGetLastError());
  b.cur ^= 1;
  return CB_OK;
}

int bits_of(uint64_t max_value) {
  int b = 1;
  while (b < 64 && (max_value >> b)) ++b;
  return b;
}

int read_u32(cb_context* ctx, const uint32_t* d, uint32_t* out) {
  CB_CUDA(cudaMemcpyAsync(out, d, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CB_CUDA(cudaStreamSynchronize(ctx->stream));
  return CB_OK;
}

Rigid rigid_of(const float* T12) { return rigid_from_t12(T12); }

// ---- accumulation over the list ---------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(kReduceBlock) pairs_pass_kernel(const IcpArgs a, const uint32_t* __restrict__ first,
                                                                  const uint32_t* __restrict__ second,
                                                                  const float* __restrict__ pair_d2, uint32_t m,
                                                                  const float* __restrict__ dst_raw,
                                                                  const float* __restrict__ dst_nrm,
                                                                  const float* __restrict__ src_raw,
                                                                  const float* __restrict__ src_nrm, const bool has_pt,
                                                                  const bool has_pl) {
  constexpr int NV = (MODE == kModeP2P || MODE == kModeP2PCentered) ? kP2PValues : kCombinedValues;
  double acc[NV];
#pragma unroll
  for (int i = 0; i < NV; i++) acc[i] = 0.0;
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < m; p += gridDim.x * blockDim.x) {
    const size_t i = first[p], j = second[p];
    const float4 dp = make_float4(dst_raw[3 * i], dst_raw[3 * i + 1], dst_raw[3 * i + 2], 0.f);
    float qx, qy, qz;
    rule::transform_point(a.T, src_raw[3 * j], src_raw[3 * j + 1], src_raw[3 * j + 2], qx, qy, qz);
    accumulate_pair<MODE>(
        acc, a, has_pt, has_pl, dp, qx, qy, qz, src_nrm != nullptr,
        [&] { return make_float4(dst_nrm[3 * i], dst_nrm[3 * i + 1], dst_nrm[3 * i + 2], 0.f); },
        [&] { return make_float4(src_nrm[3 * j], src_nrm[3 * j + 1], src_nrm[3 * j + 2], 0.f); }, pair_d2[p]);
  }
  grid_reduce<NV>(acc, a.rs);
}

}  // namespace

int launch_pairs_pass(cb_context* ctx, const IcpArgs& a, const EnginePairs& pairs, const cb_cloud* dst,
                      const cb_cloud* src, int mode, bool has_pt, bool has_pl) {
  const int blocks = std::max(1, std::min(ctx->sm_count * 4, (int)((pairs.count + kReduceBlock - 1) / kReduceBlock)));
  IcpArgs args = a;
  CB_TRY(get_reduce_scratch(ctx, blocks, kMaxValues, &args.rs));
  args.rs.ex.enabled = 0;
  ctx->pass_armed = false;
  const float* src_nrm = (mode == kModeCombined) ? src->d_raw_nrm : nullptr;
  if (mode == kModeP2PCentered)
    pairs_pass_kernel<kModeP2PCentered><<<blocks, kReduceBlock, 0, ctx->stream>>>(args, pairs.first, pairs.second, pairs.d2,
                                                                                pairs.count, dst->d_raw, dst->d_raw_nrm, src->d_raw,
                                                                                src_nrm, false, false);
  else if (mode == kModeP2P)
    pairs_pass_kernel<kModeP2P><<<blocks, kReduceBlock, 0, ctx->stream>>>(args, pairs.first, pairs.second, pairs.d2,
                                                                        pairs.count, dst->d_raw, dst->d_raw_nrm, src->d_raw, src_nrm,
                                                                        false, false);
  else
    pairs_pass_kernel<kModeCombined><<<blocks, kReduceBlock, 0, ctx->stream>>>(
        args, pairs.first, pairs.second, pairs.d2, pairs.count, dst->d_raw, dst->d_raw_nrm, src->d_raw, src_nrm, has_pt,
        has_pl);
  ctx->launches += 1;
  CB_CUDA(cudaGetLastError());
  return CB_OK;
}

int engine_find_pairs(cb_context* ctx, DeviceScope& owner, const cb_cloud* dst, const cb_cloud* src,
                      const cb_icp_params* prm, const float* T12, EnginePairs* pairs, const FeatureSet* feat) {
  // (with several ranks the caller passes the whole source cloud, replicated: capi_core.cu, ensure_src_full)
  CB_CHECK(prm->search_dir >= CB_SECOND_TO_FIRST && prm->search_dir <= CB_BOTH, CB_ERR_INVALID, "bad search_dir");
  CB_TRY(owner.free(pairs->first));
  CB_TRY(owner.free(pairs->second));
  CB_TRY(owner.free(pairs->d2));
  *pairs = EnginePairs();
  const uint32_t n_src = (uint32_t)src->n, n_dst = (uint32_t)dst->n;
  const bool want_s2f = prm->search_dir != CB_FIRST_TO_SECOND, want_f2s = prm->search_dir != CB_SECOND_TO_FIRST;
  if (n_src == 0 || n_dst == 0) return CB_OK;  // empty trees: no correspondences
  CB_TRY(ensure_index(const_cast<cb_cloud*>(dst)));
  CB_TRY(ensure_index(const_cast<cb_cloud*>(src)));
  const bool features = feat && feat->kind != CB_FEATURES_POINT;
  Dev dev(ctx);
  int *s2f_idx = nullptr, *f2s_idx = nullptr;
  float *s2f_d2 = nullptr, *f2s_d2 = nullptr;
  if (want_s2f && features) {
    // queries = transformFeatures(T) of the source features, tree = the destination features
    CB_TRY(dev.alloc(&s2f_idx, n_src));
    CB_TRY(dev.alloc(&s2f_d2, n_src));
    CB_TRY(launch_feature_nn(ctx, feat->kind, grid_view(dst), feat->dst_sorted, src->d_pts, n_src, feat->src_raw,
                             rigid_of(T12), true, prm->max_d2, s2f_idx, s2f_d2));
  } else if (want_s2f) {
    CB_TRY(dev.alloc(&s2f_idx, n_src));
    CB_TRY(dev.alloc(&s2f_d2, n_src));
    IcpArgs a;
    std::memset(&a, 0, sizeof(a));
    a.dst = grid_view(dst);
    a.src_pts = src->d_pts;
    a.n_src = n_src;
    a.T = rigid_of(T12);
    a.Tin = rigid_of(nullptr);
    a.max_d2 = prm->max_d2;
    a.out_idx = s2f_idx;
    a.out_d2 = s2f_d2;
    CB_TRY(launch_icp_pass(ctx, a, kModeKnn, true, false, false));
  }
  if (want_f2s) {
    CB_TRY(dev.alloc(&f2s_idx, n_dst));
    CB_TRY(dev.alloc(&f2s_d2, n_dst));
    cb_cloud moved(ctx, n_src, 0);  // {T src_j}: the reference's src_trans_tree_ (:201-203), rebuilt for this estimate
    CB_TRY(moved.mem.alloc(&moved.d_raw, 3 * (size_t)n_src));
    CB_TRY(launch_transform_points(ctx, rigid_of(T12), src->d_raw, n_src, moved.d_raw));
    CB_TRY(ensure_index(&moved));
    if (features) {
      // the tree over transformFeatures(T) of the source: its tails in the new grid's cell order, queried with the
      // destination features
      const Rigid T = rigid_of(T12);
      float4* moved_tails = nullptr;
      CB_TRY(dev.alloc(&moved_tails, (size_t)n_src * rule::feature_tails(feat->kind)));
      CB_TRY(launch_feature_gather(ctx, feat->kind, moved.d_pts, n_src, feat->src_raw, &T, moved_tails));
      CB_TRY(launch_feature_nn(ctx, feat->kind, grid_view(&moved), moved_tails, dst->d_pts, n_dst, feat->dst_raw,
                               rigid_of(nullptr), false, prm->max_d2, f2s_idx, f2s_d2));
    } else {
      IcpArgs a;
      std::memset(&a, 0, sizeof(a));
      a.dst = grid_view(&moved);
      a.src_pts = dst->d_pts;
      a.n_src = n_dst;
      a.T = rigid_of(nullptr);
      a.Tin = rigid_of(nullptr);
      a.max_d2 = prm->max_d2;
      a.out_idx = f2s_idx;
      a.out_d2 = f2s_d2;
      CB_TRY(launch_icp_pass(ctx, a, kModeKnn, true, false, false));
    }
  }
  // pre-filter list
  Candidates c;
  c.s2f_idx = s2f_idx;
  c.s2f_d2 = s2f_d2;
  c.f2s_idx = f2s_idx;
  c.f2s_d2 = f2s_d2;
  c.n_a = want_s2f ? n_src : 0;
  c.n_b = want_f2s ? n_dst : 0;
  c.both = prm->search_dir == CB_BOTH;
  c.reciprocal = prm->require_reciprocal != 0;
  const uint32_t total = c.n_a + c.n_b;
  PairBufs b;
  for (int k = 0; k < 2; k++) {
    CB_TRY(dev.alloc(&b.f[k], total));
    CB_TRY(dev.alloc(&b.s[k], total));
    CB_TRY(dev.alloc(&b.d[k], total));
    CB_TRY(dev.alloc(&b.keys[k], total));
    CB_TRY(dev.alloc(&b.vals[k], total));
  }
  CB_TRY(dev.alloc(&b.flags, (size_t)total + 2));
  const int nb = blocks_for(ctx, total);
  candidate_flag_kernel<<<nb, kThreads, 0, ctx->stream>>>(c, total, b.flags);
  CB_TRY(exclusive_scan_u32(ctx, b.flags, (size_t)total + 1, 0u));
  candidate_compact_kernel<<<nb, kThreads, 0, ctx->stream>>>(c, total, b.flags, b.f[0], b.s[0], b.d[0]);
  ctx->launches += 2;
  CB_CUDA(cudaGetLastError());
  uint32_t m = 0;
  CB_TRY(read_u32(ctx, b.flags + total, &m));
  const int idx_bits = bits_of(std::max(n_src, n_dst));
  // every kept value is < max_d2, and non-negative floats order like their bit patterns
  uint32_t max_bits_pattern;
  std::memcpy(&max_bits_pattern, &prm->max_d2, sizeof(uint32_t));
  const int val_bits = bits_of(max_bits_pattern);
  if (c.both) CB_TRY(sort_pairs(ctx, b, m, kKeyLex, idx_bits, idx_bits));  // lexicographic (first, second)
  // filterCorrespondencesFraction
  const double fr = prm->inlier_fraction;
  if (fr > 0.0 && fr < 1.0 && m > 0) {
    CB_TRY(sort_pairs(ctx, b, m, kKeyValuePos, val_bits, bits_of(m)));
    const long long keep = std::llround(fr * (double)m);
    m = (uint32_t)std::min<long long>(std::max<long long>(keep, 0), (long long)m);
  }
  // filterCorrespondencesOneToOne (returns early on an empty list; BOTH: no-op)
  if (prm->one_to_one && m > 0 && prm->search_dir != CB_BOTH) {
    const bool by_first = prm->search_dir == CB_SECOND_TO_FIRST;
    CB_TRY(sort_pairs(ctx, b, m, by_first ? kKeyFirstValue : kKeySecondValue, idx_bits, val_bits));
    const uint32_t* index = by_first ? b.f[b.cur] : b.s[b.cur];
    const int mb = blocks_for(ctx, m);
    group_head_flag_kernel<<<mb, kThreads, 0, ctx->stream>>>(index, m, b.flags);
    CB_TRY(exclusive_scan_u32(ctx, b.flags, (size_t)m + 1, 0u));
    flagged_compact_kernel<<<mb, kThreads, 0, ctx->stream>>>(index, m, b.flags, b.f[b.cur], b.s[b.cur], b.d[b.cur],
                                                            b.f[b.cur ^ 1], b.s[b.cur ^ 1], b.d[b.cur ^ 1]);
    ctx->launches += 2;
    CB_CUDA(cudaGetLastError());
    CB_TRY(read_u32(ctx, b.flags + m, &m));
    b.cur ^= 1;
  }
  pairs->first = b.f[b.cur];
  pairs->second = b.s[b.cur];
  pairs->d2 = b.d[b.cur];
  pairs->count = m;
  for (void* p : {(void*)pairs->first, (void*)pairs->second, (void*)pairs->d2}) dev.move_to(owner, p);
  return CB_OK;
}

}  // namespace cb
