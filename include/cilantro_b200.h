/*
 * cilantro_b200 — C ABI of the H100-native (sm_90a) rigid-ICP / k-means / RANSAC / PCA hot path.
 *
 * This is the drop-in boundary (SURVEY.md §8b). cilantro itself has no FFI: its "interface" for this
 * path is a set of C++ templates over Eigen types. Each entry point below names the reference
 * function(s) it replaces (paths relative to the reference's include/cilantro/). The header-only C++
 * shims in include/cilantro/ re-create the reference's class names on top of these calls; see
 * INTEGRATION.md for the binding a cilantro maintainer would add.
 *
 * Conventions
 *   - Plain pointers and sizes only. Host point sets are packed xyz float32, 12 B/point — exactly the
 *     memory a ConstVectorSetMatrixMap<float,3> wraps (core/data_containers.hpp:73-112,155-156).
 *   - Rigid transforms are float32[12], row-major [R | t] (3 rows of 4).
 *   - Every function returns CB_OK (0) or a negative cb_status; cb_last_error() gives the message
 *     (thread-local). Nothing throws across this boundary.
 *   - There is NO CPU fallback: without a CUDA device cb_context_create fails with CB_ERR_NO_DEVICE.
 *     Only the cb_solve_* / cb_version helpers are host-only (they are the O(1) 3x3 / 6x6 solves the
 *     reference also runs on the host).
 *   - One cb_context per (process, device); calls on one context are serialised by the caller,
 *     like the reference's objects (not thread-safe, SURVEY.md §8b "Threading").
 */
#ifndef CILANTRO_B200_H_
#define CILANTRO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default) /* the library is built with -fvisibility=hidden */
#endif

typedef enum cb_status {
  CB_OK = 0,
  CB_ERR_INVALID = -1,    /* bad argument */
  CB_ERR_NO_DEVICE = -2,  /* no usable CUDA device / driver */
  CB_ERR_CUDA = -3,       /* CUDA runtime error (message in cb_last_error) */
  CB_ERR_NCCL = -4,       /* NCCL missing or failed */
  CB_ERR_UNSUPPORTED = -5
} cb_status;

typedef struct cb_context cb_context;
typedef struct cb_cloud cb_cloud;
typedef struct cb_vectors cb_vectors;
typedef struct cb_icp cb_icp;

const char* cb_last_error(void);
const char* cb_version(void);

/* ---- context -------------------------------------------------------------------------------- */
int cb_context_create(int device, cb_context** out);
void cb_context_destroy(cb_context* ctx);
int cb_context_synchronize(cb_context* ctx);
/* SM count, total HBM bytes of the context's device. */
int cb_context_device_info(cb_context* ctx, int* sm_count, size_t* hbm_bytes, char* name64);
/* Number of kernels this library has launched on the context since creation (for bench.py's
 * gpu_launches claim). */
uint64_t cb_context_kernel_launches(cb_context* ctx);
/* Evict L2 by writing a scratch buffer larger than L2 (bench hygiene; not part of any algorithm). */
int cb_context_flush_l2(cb_context* ctx);

/* Multi-GPU: one process per GPU. Rank 0 calls cb_comm_unique_id, the 128 bytes are broadcast by
 * the launcher's own channel (torch.distributed in bench.py), every rank calls cb_context_init_comm.
 * Afterwards ICP / k-means / PCA objects created from shards on this context reduce their normal
 * equations / centroid sums across ranks with ONE ncclAllReduce per iteration (SURVEY.md §8e).
 * The reference has no counterpart (single process, OpenMP reductions:
 * core/openmp_reductions.hpp:3-33, registration/transform_estimation.hpp:285-290). */
int cb_comm_unique_id(void* out_128_bytes);
int cb_context_init_comm(cb_context* ctx, const void* unique_id_128_bytes, int rank, int world);
int cb_context_comm_info(cb_context* ctx, int* rank, int* world);
/* Optional, after cb_context_init_comm: the FUSED exchange. Every rank exports a 64-byte CUDA-IPC
 * handle of its exchange table (cb_comm_ipc_handle), the launcher all-gathers them in rank order
 * (world x 64 bytes) and every rank maps its peers' tables (cb_comm_ipc_attach), then barriers.
 * From then on the ICP accumulation kernel itself all-reduces the 16/28 moments by writing them
 * straight into the peers' tables over NVLink and publishes the total to a mapped host mailbox, so an
 * iteration costs one kernel + one host poll: no ncclAllReduce, cudaMemcpy or stream synchronise.
 * If mapping fails (no peer access) the call returns an error and the NCCL path stays active. */
int cb_comm_ipc_handle(cb_context* ctx, void* out_64_bytes);
int cb_comm_ipc_attach(cb_context* ctx, const void* handles_world_x_64_bytes);
/* Back to the NCCL reduction on this rank. The launcher calls it on EVERY rank when cb_comm_ipc_attach failed
 * on any of them (the ranks must agree on the path before the first pass). */
int cb_comm_ipc_detach(cb_context* ctx);

/* ---- device-resident point sets --------------------------------------------------------------
 * Replaces: PointFeaturesAdaptor<float,3> ctor (correspondence_search/
 * common_transformable_feature_adaptors.hpp:14-17) for query sets, and the KDTree<float,3> ctor
 * (core/kd_tree.hpp:162-170 -> nanoflann buildIndex) for reference sets: the points are uploaded
 * once, binned into a uniform grid (cell-sorted float4 copy + cell-start table) and stay in HBM.
 * normals may be NULL. index_offset is added to this set's point indices in every result
 * (a rank's shard offset; 0 on a single GPU). */
int cb_cloud_create(cb_context* ctx, const float* xyz, const float* normals, size_t n, uint64_t index_offset,
                    cb_cloud** out);
/* Two clouds in one call — what the constructors of the ICP classes receive (icp_common_instances.hpp:34-44:
 * dst points [+ normals], src points [+ normals]). Same result as two cb_cloud_create calls followed by the lazy
 * index builds, but the upload of the second cloud runs on a second stream while the grid of the first is being
 * built (effective with pinned host buffers). Both clouds are indexed on return. */
int cb_cloud_create_pair(cb_context* ctx, const float* xyz_a, const float* normals_a, size_t n_a, uint64_t offset_a,
                         const float* xyz_b, const float* normals_b, size_t n_b, uint64_t offset_b, cb_cloud** out_a,
                         cb_cloud** out_b);
/* Same, from packed xyz already in device memory (used when inputs are HBM-resident). */
int cb_cloud_create_from_device(cb_context* ctx, const float* d_xyz, const float* d_normals, size_t n,
                                uint64_t index_offset, cb_cloud** out);

/* Multi-rank: a cloud EVERY rank needs in full (the replicated destination cloud of a sharded ICP —
 * SURVEY 8e) built from its contiguous blocks: each rank uploads only block [first_index, first_index + n_block) of the
 * n_total points over its own PCIe link, the blocks are exchanged over NVLink (NCCL) and every rank ends up with the
 * same cloud as cb_cloud_create(whole array) would give it, bit for bit. Collective over the context's communicator
 * (cb_context_init_comm); with world == 1 it is cb_cloud_create. Normals: present on all ranks or on none. */
int cb_cloud_create_replicated(cb_context* ctx, const float* xyz_block, const float* normals_block, size_t n_block,
                               uint64_t first_index, size_t n_total, cb_cloud** out);
void cb_cloud_destroy(cb_cloud* c);
size_t cb_cloud_size(const cb_cloud* c);
/* Grid facts for DESIGN/bench reporting: cell edge, dims[3], occupied-cell mean occupancy. */
int cb_cloud_grid_info(const cb_cloud* c, float* cell_edge, int* dims3, double* mean_occupancy);

/* ---- nearest neighbour ------------------------------------------------------------------------
 * cb_knn1_radius replaces the batched KDTree::kNNInRadiusSearch(q, k=1, r2) sweep of
 * findNNCorrespondencesUnidirectional (correspondence_search/
 * correspondence_search_kd_tree_utilities.hpp:26-33 -> core/kd_tree.hpp:284-291) with the query
 * transform of PointFeaturesAdaptor::transformFeatures fused in (T may be NULL = identity).
 * For query i (original order): idx[i] = index of the nearest ref point with d2 < max_d2 (lowest
 * index on exact ties), or -1; d2[i] = its squared distance, or max_d2.
 * max_d2 = FLT_MAX gives KDTree::nearestNeighborSearch (core/kd_tree.hpp:181-204). */
int cb_knn1_radius(cb_context* ctx, const cb_cloud* ref, const cb_cloud* qry, const float* T12, float max_d2,
                   int64_t* idx, float* d2);
/* General k (1..256; CB_ERR_UNSUPPORTED above): KDTree::kNNInRadiusSearch / kNNSearch batched (core/kd_tree.hpp:215-318).
 * idx/d2 are n_qry x k, ascending d2, unused slots idx = -1. counts (may be NULL) = found per query. */
int cb_knn_radius(cb_context* ctx, const cb_cloud* ref, const cb_cloud* qry, const float* T12, int k,
                  float max_d2, int64_t* idx, float* d2, uint32_t* counts);
/* KDTree::radiusSearch batched (core/kd_tree.hpp:250-278): for query i, every ref point with d2 < radius2,
 * ascending d2 (equal distances: ascending index; the reference leaves them to std::sort), as a CSR list:
 * entries offsets[i] .. offsets[i+1]-1 of idx / d2; offsets has n_qry + 1 entries. *total = offsets[n_qry].
 * Sizing: call with idx = d2 = NULL (or a too small capacity) -> offsets and *total are filled, nothing else
 * is written; call again with buffers of capacity >= *total. */
int cb_radius_search(cb_context* ctx, const cb_cloud* ref, const cb_cloud* qry, const float* T12, float radius2,
                     uint64_t* offsets, int64_t* idx, float* d2, size_t capacity, size_t* total);
/* ---- normal / curvature estimation -------------------------------------------------------------
 * Replaces NormalEstimation::estimateNormalsAndCurvature{KNN,Radius,KNNInRadius} (core/
 * normal_estimation.hpp:83-232 -> compute_normals_curvature_* :357-421) as called by
 * PointCloud::estimateNormals* (utilities/point_cloud.hpp:294-420). Neighbourhood of every point over
 * the cloud itself:  k > 0, radius2 <= 0 : kNN;  k > 0, radius2 > 0 : kNN within squared radius;
 * k == 0, radius2 > 0 : all points with d2 < radius2 (cilantro radii are squared distances).
 * Fewer than 3 neighbours -> NaN. view_point3 (may be NULL or non-finite = no orientation step) flips
 * each normal towards the view point (:325-329); use_current_as_ref != 0 on a cloud that has normals
 * orients by those instead (setReferenceNormals, :63-69, :351-355; takes precedence, :281-291). The normals are stored in the cloud on the device (as
 * PointCloud::normals is filled), so a combined-metric ICP can follow without a host round trip.
 * Host outputs (each may be NULL): normals 3n, curvature n, cov6 6n (xx,xy,xz,yy,yz,zz of the
 * neighbourhood covariance, diagnostic). gpu_ms (may be NULL) = device time of the kernel. k <= 128
 * (the k-best lists live in shared memory; CB_ERR_UNSUPPORTED above). */
int cb_cloud_estimate_normals(cb_context* ctx, cb_cloud* cloud, int k, float radius2, const float* view_point3,
                              int use_current_as_ref, float* normals, float* curvature, float* cov6, float* gpu_ms);

/* ---- robust normal estimation (minimum covariance determinant) ---------------------------------
 * Replaces NormalEstimation<float, 3, MinimumCovarianceDeterminant<float, 3>> (core/normal_estimation.hpp:279-421
 * over MinimumCovarianceDeterminant::operator(), core/covariance.hpp:185-371). Per point, over its neighbourhood
 * (size m, in ascending (d2, index) order): m < min_sample_size -> invalid; m == min_sample_size -> the plain
 * covariance; else h = min(max(min_sample_size, llround(inlier_ratio * m)), m); h == m -> the plain covariance (bit
 * for bit cb_cloud_estimate_normals'); else num_trials trials of min_sample_size draws with replacement, each refined
 * num_refinements times (keep the h smallest Mahalanobis distances, recompute), and the trial of smallest finite
 * determinant wins. With chi_square_threshold > 0, the neighbourhood's first point must lie within d_M^2 <= threshold.
 * Normal, curvature and orientation then follow cb_cloud_estimate_normals. The random draws, the selection order
 * and the 3x3 algebra follow the rule of DESIGN §4.15 (cilantro_b200/csrc/mcd_rule.hpp): every point runs
 * std::minstd_rand0 seeded from `seed` and its index, so equal seeds give equal bits.
 * Neighbourhoods: k in [1, 128], kNN (radius2 <= 0) or kNN-in-radius (radius2 > 0); radius-only (k == 0) gives
 * CB_ERR_UNSUPPORTED. Rejected: num_trials < 1, num_refinements < 0 or a non-finite inlier_ratio (CB_ERR_INVALID);
 * min_sample_size outside [2, 32] or k > 128 (CB_ERR_UNSUPPORTED). Outputs as cb_cloud_estimate_normals', plus
 * status (n bytes, may be NULL): 0 ok, 1 too few neighbours, 2 rejected by the chi-square test, 3 no trial with a
 * finite determinant; every status but 0 gives NaN normal, curvature and cov6. */
typedef struct cb_mcd_params {
  int num_trials;             /* 6 in the reference */
  int num_refinements;        /* 3 */
  float inlier_ratio;         /* 0.75 */
  float chi_square_threshold; /* -1: no test */
  int min_sample_size;        /* 3 (NormalEstimation's setMinValidSampleSize(3)) */
  uint32_t seed;              /* replaces the reference's std::random_device */
} cb_mcd_params;
int cb_cloud_estimate_normals_mcd(cb_context* ctx, cb_cloud* cloud, int k, float radius2, const float* view_point3,
                                  int use_current_as_ref, const cb_mcd_params* params, float* normals, float* curvature,
                                  float* cov6, uint8_t* status, float* gpu_ms);
/* ---- voxel-grid downsampling -------------------------------------------------------------------
 * Replaces PointCloud::gridDownsample / gridDownsampled (utilities/point_cloud.hpp:246-290) =
 * Points[Normals][Colors]GridDownsampler (core/grid_downsampler.hpp) over GridAccumulator::build_index_
 * (core/grid_accumulator.hpp:146-199): bin = floor(p * (1 / bin_size)) per axis; per bin the point sum,
 * the sign-consistent normal sum (core/common_accumulators.hpp:122-131) and the colour sum are taken
 * in point-index order in fp32 (the serial build's arithmetic, bit for bit) and divided by the count;
 * normals are re-normalised; bins with fewer than min_points_in_bin points are dropped.
 * order = 0: bins ascending lexicographically in (x, y, z) — the std::map order the default
 *            (parallel = true) build emits (:177-181);
 * order = 1: bins in order of their first point — the serial (parallel = false) build (:194-197).
 * normals / colors (packed 3 floats per point) may be NULL; outputs are sized for n points, *out_n is
 * the number of occupied bins written. */
int cb_grid_downsample(cb_context* ctx, const float* xyz, const float* normals, const float* colors, size_t n,
                       float bin_size, size_t min_points_in_bin, int order, float* out_xyz, float* out_normals,
                       float* out_colors, size_t* out_n);
/* Same on a device-resident cloud (points + normals if it has them); the result is a new cloud that never
 * leaves HBM (downsample -> cb_cloud_estimate_normals -> cb_icp_* without host round trips). gpu_ms may be
 * NULL. */
int cb_cloud_grid_downsample(cb_context* ctx, const cb_cloud* cloud, float bin_size, size_t min_points_in_bin,
                             int order, cb_cloud** out, float* gpu_ms);
/* ---- connected-component segmentation ----------------------------------------------------------
 * Replaces ConnectedComponentExtraction3f::segment(nh, [seeds,] evaluator, min, max) (clustering/
 * connected_component_extraction.hpp:368-428) = extractConnectedComponents over a kd-tree (:163-265, the same logic
 * as the neighbourhood-set form :21-118), restated for one thread (the reference's OpenMP seed loop is not
 * reproducible, DESIGN §6). For point p, N(p) = its neighbourhood over the cloud, ascending (d2, index) — the lists
 * cb_knn_radius / cb_radius_search return; the encoding is cb_cloud_estimate_normals': k > 0, radius2 <= 0: kNN;
 * k > 0, radius2 > 0: kNN within radius2; k == 0, radius2 > 0: all points with d2 < radius2. Edge p -> q iff q is at
 * position >= 1 of N(p) (`for j = 1`, :201) and the evaluator accepts (p, q, d2). Labelled = reachable from the
 * seeds (seeds == NULL: every point; n_seeds == 0 with a non-NULL pointer: none); segments = weakly connected
 * components of the labelled points; segments with fewer than min or more than max points are dropped (:246-261);
 * order = size descending, equal sizes by the smallest seed-list position of a seed in the segment (all seeds: the
 * smallest point index), which is what std::stable_sort gives where :263 uses std::sort; points ascending.
 * Evaluator (core/common_pair_evaluators.hpp:88-259; terms combined with AND, 0 = AlwaysTrueEvaluator):
 *   CB_SEG_POINTS   d2 < max_distance (max_distance is compared with the SQUARED distance, like the reference)
 *   CB_SEG_NORMALS  acosf(ni . nj) <= max_angle (< when angle_strict, as in the combined evaluators); max_angle < 0:
 *                   min(angle, pi - angle) against -max_angle (unoriented normals)
 *   CB_SEG_COLORS   |ci - cj|^2 < max_color_diff2 (the evaluators square the threshold in fp32 in their constructor)
 * normals: host array (3n) or NULL = the normals stored in the cloud (cb_cloud_create / cb_cloud_estimate_normals);
 * colors: host array (3n), required with CB_SEG_COLORS. Outputs, sized by n: point_to_cluster[n] (unlabelled =
 * *num_clusters, clustering_base.hpp:8-17), cluster_offsets[*num_clusters + 1], cluster_points[offsets[last]] (CSR of
 * getClusterToPointIndicesMap). Single GPU: a cloud with index_offset != 0 gives CB_ERR_UNSUPPORTED; k <= 256. Seeds
 * out of range, or a missing normals / colors array: CB_ERR_INVALID. gpu_ms (may be NULL) = device time. */
typedef enum cb_segment_term { CB_SEG_POINTS = 1, CB_SEG_NORMALS = 2, CB_SEG_COLORS = 4 } cb_segment_term;
typedef struct cb_segment_params {
  int32_t k;
  float radius2;
  int32_t terms;         /* cb_segment_term bits */
  int32_t angle_strict;  /* 0: NormalsProximityEvaluator (<=); 1: the combined evaluators (<) */
  float max_distance;
  float max_angle;       /* radians */
  float max_color_diff2;
  int32_t reserved_;
  uint64_t min_segment_size;
  uint64_t max_segment_size;
} cb_segment_params;
int cb_cloud_segment(cb_context* ctx, cb_cloud* cloud, const cb_segment_params* params, const float* normals,
                     const float* colors, const uint64_t* seeds, size_t n_seeds, uint64_t* point_to_cluster,
                     uint64_t* cluster_offsets, uint64_t* cluster_points, size_t* num_clusters, float* gpu_ms);
/* ---- mean-shift clustering ---------------------------------------------------------------------
 * Replaces MeanShift3f::cluster(seeds, kernel_radius, max_iter, cluster_tol, convergence_tol, evaluator)
 * (clustering/mean_shift.hpp:37-115) and the all-points overload (:118-124, seeds == NULL: the cloud's own points).
 * Shift (:45-82): r2 = kernel_radius^2 (kernel_radius is a distance, not a squared one), tol2 = convergence_tol^2;
 * every iteration, every seed not yet converged takes N = the cloud points with d2 < r2, ascending (d2, index) (the
 * reference leaves equal distances to std::sort), sums acc += w p_j and W += w in that order in fp32,
 * m = acc * (1 / W), is marked converged when |seed - m|^2 < tol2, and becomes m. The loop stops after the first
 * iteration whose processed seeds all converged, or at max_iter (zero seeds: 1 iteration). A seed without
 * neighbours becomes NaN (0 * inf) and never converges. Cluster (:84-100): seed i joins the first cluster, in
 * creation order, whose first seed is within |.|^2 < cluster_tol^2, else starts one. Modes (:102-112): the fp32 sum
 * of the members' shifted seeds in member order times 1 / size.
 * Weight (cb_weight_kind): CB_WEIGHT_UNITY (UnityWeightEvaluator, the default) or CB_WEIGHT_RBF
 * (RBFKernelWeightEvaluator<float, float, true>: exp(weight_coeff * d2), weight_coeff = -0.5f / (sigma * sigma)).
 * Outputs, sized by n_seeds: shifted_seeds[3 n_seeds], point_to_cluster[n_seeds] (indexed by SEED),
 * cluster_offsets[n_seeds + 1], cluster_points[n_seeds] (CSR of getClusterToPointIndicesMap, seeds ascending),
 * modes[3 n_seeds] (the first *num_clusters rows are written); *iterations = getNumberOfPerformedIterations().
 * A cloud with index_offset != 0 or more than 2^31 - 1 seeds: CB_ERR_UNSUPPORTED; an empty cloud with seeds:
 * CB_ERR_INVALID (the reference's kd-tree throws on an empty index); the seed limit is 2^31 - 1 because seed ids travel as
 * 32-bit signed slots through the radius-list kernels. gpu_ms (may be NULL) = device time of the call, gpu_ms_shift
 * (may be NULL) = the part spent in the shift loop (the rest is the clustering and the modes). */
typedef struct cb_mean_shift_params {
  float kernel_radius;
  int32_t weight_kind;   /* cb_weight_kind */
  uint64_t max_iter;
  float cluster_tol;
  float convergence_tol; /* FLT_EPSILON in the reference's signature */
  float weight_coeff;    /* CB_WEIGHT_RBF only */
  int32_t reserved_;
} cb_mean_shift_params;
int cb_cloud_mean_shift(cb_context* ctx, cb_cloud* cloud, const cb_mean_shift_params* params, const float* seeds,
                        size_t n_seeds, float* shifted_seeds, uint64_t* point_to_cluster, uint64_t* cluster_offsets,
                        uint64_t* cluster_points, float* modes, size_t* num_clusters, uint64_t* iterations,
                        float* gpu_ms, float* gpu_ms_shift);
/* Copies a cloud's points (and normals, if normals != NULL and the cloud has them) back to the host in
 * original order. */
int cb_cloud_download(cb_context* ctx, const cb_cloud* cloud, float* xyz, float* normals);
/* findNNCorrespondencesUnidirectional(ref_is_first = true), compacted in query order:
 * (index_first[c], index_second[c], value[c]) = (ref idx, query idx, d2). Arrays sized n_qry. */
int cb_find_correspondences(cb_context* ctx, const cb_cloud* ref, const cb_cloud* qry, const float* T12,
                            float max_d2, uint64_t* index_first, uint64_t* index_second, float* value,
                            size_t* count);

/* ---- rigid ICP -------------------------------------------------------------------------------
 * cb_icp_* replaces SimplePointToPointMetricRigidICP3f / SimpleCombinedMetricRigidICP3f
 * (registration/icp_common_instances.hpp:34-97,250,261): IterativeClosestPointBase::estimate()
 * (registration/icp_base.hpp:68-87) with, per iteration, ONE fused kernel doing
 *   transformFeatures (common_transformable_feature_adaptors.hpp:28-34)
 * + the radius-bounded 1-NN sweep (correspondence_search_kd_tree_utilities.hpp:26-33)
 * + transformPoints (core/space_transformations.hpp:203-216)
 * + the normal-equation / Kabsch-moment accumulation
 *   (registration/transform_estimation.hpp:25-34, :298-343, :669-715),
 * then one small all-reduce when a communicator is attached, then the host-side solve
 * (transform_estimation.hpp:36-45, :346-357; core/space_transformations.hpp:43-51). */
typedef enum cb_icp_metric {
  CB_ICP_POINT_TO_POINT = 0, /* PointToPointMetricSingleTransformICP (Kabsch per iteration) */
  CB_ICP_COMBINED = 1        /* CombinedMetricSingleTransformICP; symmetric if src has normals */
} cb_icp_metric;

typedef struct cb_icp_params {
  int32_t metric;
  int32_t max_iter;     /* icp_base.hpp:24, default 15 */
  float tol;            /* icp_base.hpp:25, default 1e-5 */
  float max_d2;         /* SQUARED; correspondence_search_kd_tree.hpp:49, default 0.01*0.01 */
  float w_pt;           /* icp_single_transform_combined_metric.hpp:46, default 0 */
  float w_pl;           /* :47, default 1 */
  int32_t max_opt_iter; /* :44, default 1 */
  float opt_tol;        /* :45, default 1e-5 */
  float T_init[12];     /* icp_base.hpp:58-61 */
  int32_t flush_l2;     /* bench hygiene: evict L2 before every iteration (outside the timed events) */
  int32_t timing;       /* CUDA-event instrumentation of estimate(): 0 none (production), 1 one bracket per
                           iteration (kernel + exchange + host solve) -> gpu_ms_total / cb_icp_iteration_times,
                           2 one bracket per search kernel -> gpu_ms_search. Each cudaEventRecord costs a few us of
                           device front-end time, comparable to the ~100 us iteration, hence one mode at a time. */
  /* Correspondence-engine options (correspondence_search_kd_tree.hpp:46-50, :60-98 setters). The defaults
   * (SECOND_TO_FIRST, fraction 1, no reciprocity, not one-to-one) take the fused single-kernel path; any other
   * setting materialises the correspondence list on the device (search(es) -> union / intersection -> fraction
   * filter -> one-to-one filter, core/correspondence.hpp:57-100) and accumulates over it. With several ranks every rank runs
   * them on the whole source cloud (shards all-gathered once; create the shards with index_offset = their first global index):
   * same lists and transforms as one GPU, on every rank. */
  int32_t search_dir;          /* cb_search_dir; default CB_SECOND_TO_FIRST */
  int32_t require_reciprocal;  /* with CB_BOTH: intersection instead of union (:68-70 of ..._utilities.hpp) */
  int32_t one_to_one;          /* keep, per dst (SECOND_TO_FIRST) / src (FIRST_TO_SECOND) point, the closest pair */
  int32_t host_loop;           /* 0 (default): iterations run back to back on the device where the configuration allows it
                                  (default engine, one Gauss-Newton step per iteration); 1: host-driven loop (A/B, tests) */
  double inlier_fraction;      /* keep the llround(fraction * M) closest pairs when 0 < fraction < 1; default 1 */
  /* Correspondence weight evaluators of the combined / symmetric metric (the PointToPointCorrWeightEvaluatorT /
   * PointToPlaneCorrWeightEvaluatorT template arguments of CombinedMetricSingleTransformICP, consumed at
   * registration/transform_estimation.hpp:302-304 and :331-333): weight = metric weight * evaluator(i, j, d2).
   * Arbitrary functors cannot cross a C ABI; the two evaluators of core/common_pair_evaluators.hpp that make sense
   * here are selected by kind: CB_WEIGHT_UNITY (UnityWeightEvaluator, :29-43, the default) and CB_WEIGHT_RBF
   * (RBFKernelWeightEvaluator<float, float, true>, :46-79: exp(coeff * d2) with coeff = -0.5f / (sigma * sigma),
   * d2 = the correspondence's squared distance). */
  int32_t pt_weight_kind;
  int32_t pl_weight_kind;
  float pt_weight_coeff;
  float pl_weight_coeff;
} cb_icp_params;

typedef enum cb_weight_kind { CB_WEIGHT_UNITY = 0, CB_WEIGHT_RBF = 1 } cb_weight_kind;

typedef enum cb_search_dir {
  CB_SECOND_TO_FIRST = 0, /* queries = transformed src, tree = dst (the default) */
  CB_FIRST_TO_SECOND = 1, /* queries = dst, tree = transformed src (rebuilt every iteration) */
  CB_BOTH = 2
} cb_search_dir;

typedef struct cb_icp_result {
  float T[12];
  int32_t iterations;
  float last_delta;
  int32_t converged;
  uint64_t num_corr;    /* correspondences of the last iteration (global across ranks) */
  double gpu_ms_total;  /* sum over iterations of the CUDA-event time of the iteration's kernels */
  double gpu_ms_search; /* ... of which the fused search+accumulate kernel */
  uint64_t kernel_launches;
} cb_icp_result;

void cb_icp_default_params(cb_icp_params* p);
/* dst must carry normals for CB_ICP_COMBINED. Both clouds must outlive the icp object. */
int cb_icp_create(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src, cb_icp** out);
void cb_icp_destroy(cb_icp* icp);
int cb_icp_estimate(cb_icp* icp, const cb_icp_params* prm, cb_icp_result* res);
/* Per-iteration device times of the last estimate() (ms); n = min(cap, iterations). */
int cb_icp_iteration_times(cb_icp* icp, double* ms, int cap);
/* getCorrespondences() of the engine after the last iteration (this rank's shard). Arrays hold n_src entries
 * (n_src + n_dst when search_dir == CB_BOTH). Default mode: ascending source index; other engine modes: the
 * order the reference's filters leave (ascending value after the fraction filter, ascending dst / src index
 * after the one-to-one filter, lexicographic (first, second) for CB_BOTH). */
int cb_icp_correspondences(cb_icp* icp, uint64_t* index_first, uint64_t* index_second, float* value,
                           size_t* count);
/* computeResiduals() — icp_single_transform_combined_metric.hpp:220-243 /
 * icp_single_transform_point_to_point_metric.hpp:68-85. out has n_src floats (this rank's shard). */
int cb_icp_residuals(cb_icp* icp, const cb_icp_params* prm, const float* T12, float* out);

/* One fused search+accumulate pass WITHOUT the solve: returns the reduced moments.
 * p2p: sums[16] = {n, sum d (3), sum q (3), sum d q^T (9, row-major)}
 * combined: sums[28] = {n, AtA upper triangle row-major (21), Atb (6)}. Used by the parity tests
 * and by callers that do their own reduction. */
int cb_icp_accumulate(cb_icp* icp, const cb_icp_params* prm, const float* T12, double* sums, int cap);

/* Inspection of the device-resident loop's per-query cache after cb_icp_estimate took that path (parity tests):
 * T_search12 = the transform the LAST executed iteration searched with; nearest[i] = original index of the
 * destination point the loop holds as source point i's nearest neighbour under that transform (whether or not it
 * is inside the radius), -1 = none known; searched_last = queries the last iteration had to search again.
 * Returns CB_ERR_INVALID when the last estimate() did not run on the device loop. */
int cb_icp_loop_cache(cb_icp* icp, float* T_search12, int64_t* nearest, uint64_t* searched_last);

/* Feature-space correspondence search: CorrespondenceSearchKDTree<SearchFeatureAdaptorT> over the feature adaptors of
 * correspondence_search/common_transformable_feature_adaptors.hpp, as CombinedMetricRigidTransformICP3f<Engine> /
 * PointToPointMetricRigidTransformICP3f<Engine> take it (registration/icp_single_transform_combined_metric.hpp:262-267,
 * icp_single_transform_point_to_point_metric.hpp:96-98):
 *   CB_FEATURES_POINT               [p]                  PointFeaturesAdaptor3f (the default: xyz only)
 *   CB_FEATURES_POINT_NORMAL        [p, w_n n]           PointNormalFeaturesAdaptor3f
 *   CB_FEATURES_POINT_COLOR         [p, w_c c]           PointColorFeaturesAdaptor3f
 *   CB_FEATURES_POINT_NORMAL_COLOR  [p, w_n n, w_c c]    PointNormalColorFeaturesAdaptor3f
 * The arrays are host n x 3 (destination / source cloud order), copied and weighted at this call; the ones a kind
 * does not use may be NULL. They are separate from the clouds' normals: source normals on the cloud make the metric
 * symmetric, a feature adaptor does not. The source features are transformed with the estimate as transformFeatures
 * does (normal part rotated, colour part copied). The correspondence search then runs on the feature distance (the
 * correspondence value, the radius test, the weight evaluators and the engine filters all see the feature d2), while
 * the estimator uses the 3-D points and destination normals as before; cb_icp_residuals stays a 3-D search, as the
 * reference's computeResiduals. Every other kind than CB_FEATURES_POINT takes the list path of the non-default engine
 * modes, whatever cb_icp_params says; CB_FEATURES_POINT drops the features and restores the default paths.
 * CB_ERR_INVALID: an array the kind needs is NULL, or a weight the kind uses is not finite. Several ranks:
 * CB_ERR_UNSUPPORTED. */
typedef enum cb_feature_kind {
  CB_FEATURES_POINT = 0,
  CB_FEATURES_POINT_NORMAL = 1,
  CB_FEATURES_POINT_COLOR = 2,
  CB_FEATURES_POINT_NORMAL_COLOR = 3
} cb_feature_kind;
int cb_icp_set_features(cb_icp* icp, int kind, const float* dst_normals, const float* dst_colors,
                        const float* src_normals, const float* src_colors, float normal_weight, float color_weight);

/* Projective correspondence search: CorrespondenceSearchProjective<float> as SimpleCombinedMetricRigidProjectiveICP3f
 * and the ICPs over that engine take it (correspondence_search/correspondence_search_projective.hpp:156-209). K9 is the
 * row-major 3 x 3 intrinsic matrix, w x h the image, E12 the row-major 3 x 4 camera pose [R | t] (NULL = identity).
 * This call builds the index map over the destination cloud (pointsToIndexMap's rule: smallest camera z, lowest index
 * on ties, non-finite points skipped) and keeps it on the device, 4 B per pixel, until the next call or
 * cb_icp_destroy. From then on every source point q = T s is matched to the destination point its pixel
 * (llround of the projection through E^-1 and K) shows, kept iff its squared distance is < max_d2; the list is in
 * ascending source index and a destination point may be matched many times (DESIGN §4.21). cb_icp_estimate,
 * cb_icp_accumulate and cb_icp_correspondences honour it, with inlier_fraction < 1 applied as
 * filterCorrespondencesFraction; cb_icp_residuals stays the kd-tree search, as the reference's computeResiduals;
 * cb_icp_loop_cache returns CB_ERR_INVALID after a projective run. K9 = NULL detaches the projection and restores the
 * kd-tree paths. w or h = 0: no correspondences. CB_ERR_INVALID: non-finite K9 or E12, w h >= 2^32, and at
 * cb_icp_estimate / cb_icp_accumulate a search_dir other than CB_SECOND_TO_FIRST, require_reciprocal, one_to_one or
 * features attached. Several ranks: CB_ERR_UNSUPPORTED. On an error the projection attached before the call (or none)
 * stays in force. Launches: 3 (2 for an empty destination cloud). */
int cb_icp_set_projection(cb_icp* icp, const float* K9, size_t w, size_t h, const float* E12);

/* Host-only O(1) solves (no device needed; exported so the N>1 logic is testable on CPU). */
/* estimateTransformPointToPointMetric from moments — transform_estimation.hpp:25-47. Returns 1 if n>=3. */
int cb_solve_kabsch_moments(const double* sums16, float* T12);
/* Symmetric eigen-decomposition of the D x D row-major A in fp64 (Householder + implicit symmetric QR), the solve of
 * PrincipalComponentAnalysis::compute_ (principal_component_analysis.hpp:76-84): evals descending, evecs row-major with
 * unit eigenvector columns, each signed so that its largest-magnitude component is positive (lowest index on ties),
 * then the last column negated if det < 0. Returns 1; 0 for a non-finite A (all-NaN output); CB_ERR_UNSUPPORTED
 * (all-NaN output) when the QR iteration does not converge, which cb_vectors_pca reports the same way. */
int cb_solve_sym_eigen(const double* A, int D, float* evals, float* evecs);
/* One Gauss-Newton update of estimateTransformCombinedMetric — :346-357: T_out = Ra ta Ra T_in. */
int cb_solve_gauss_newton(const double* sums28, const float* T_in12, float* T_out12, float* dtheta_norm);
/* LinearTransform::rotation() — core/space_transformations.hpp:43-51 (3x3 row-major in/out). */
int cb_solve_rotation(const float* L9, float* R9);
/* tform_iter * transform_ and the update norm — icp_single_transform_combined_metric.hpp:213-216. */
int cb_compose(const float* A12, const float* B12, float* out12);

/* ---- k-means ---------------------------------------------------------------------------------
 * Replaces KMeans<float,3>::cluster(centroids, max_iter, tol, use_kd_tree=false)
 * (clustering/kmeans.hpp:24-30,67-194): fused brute-force assignment (:100-119) + per-cluster
 * sums (:126-131) in one kernel, one all-reduce of K x 4 sums when a communicator is attached,
 * empty-cluster repair (:134-176) and the division (:179-181) on the host.
 * centroids: in = initial (K x 3), out = final. labels (may be NULL): n uint64, ORIGINAL order. */
typedef struct cb_kmeans_result {
  uint64_t iterations;
  double gpu_ms_total;
  uint64_t kernel_launches;
} cb_kmeans_result;
int cb_kmeans_cluster(cb_context* ctx, const cb_cloud* pts, float* centroids, size_t k, size_t max_iter,
                      float tol, uint64_t* labels, cb_kmeans_result* res);
/* One assignment sweep against given centroids (kmeans.hpp:100-119); labels n uint64. Also returns
 * the per-cluster sums (K x 3 doubles) and counts (K uint64) when non-NULL. */
int cb_kmeans_assign(cb_context* ctx, const cb_cloud* pts, const float* centroids, size_t k, uint64_t* labels,
                     double* sums, uint64_t* counts);
/* KMeans::cluster(num_clusters,...) seeding (kmeans.hpp:32-49) with an injected seed. */
int cb_kmeans_seed_indices(size_t n, size_t k, uint32_t seed, uint64_t* out_idx);

/* ---- D-dimensional vector sets and k-means over them -------------------------------------------
 * A cb_vectors holds n x D float32 rows in HBM, point-major: the bytes a ConstVectorSetMatrixMap<float, D>
 * (core/data_containers.hpp:73-112) wraps. D >= 1; D <= 0 or a null pointer is CB_ERR_INVALID, except a null data
 * pointer with n = 0 (an empty set, as for clouds). */
int cb_vectors_create(cb_context* ctx, const float* data, size_t n, int D, cb_vectors** out);
int cb_vectors_create_from_device(cb_context* ctx, const float* d_data, size_t n, int D, cb_vectors** out);
void cb_vectors_destroy(cb_vectors* v);
size_t cb_vectors_size(const cb_vectors* v);
/* KMeans<float, D, KDTreeDistanceAdaptors::L2>::cluster(centroids, max_iter, tol, use_kd_tree=false)
 * (clustering/kmeans.hpp:9-59,67-194, brute-force branch) for any D: cb_kmeans_cluster over D-dimensional rows,
 * with the distance d = c - p, acc = d[D-1]^2, acc = d[j]^2 + acc for j = D-2 .. 0 (fp32, no FMA; at D = 3 it is
 * cb_kmeans_cluster's). centroids: in = initial (k x D), out = final. labels (may be NULL): n uint64. One GPU: a
 * context with several ranks returns CB_ERR_UNSUPPORTED. */
int cb_kmeans_cluster_vectors(cb_context* ctx, const cb_vectors* vectors, float* centroids, size_t k, size_t max_iter,
                              float tol, uint64_t* labels, cb_kmeans_result* res);
/* One assignment sweep (kmeans.hpp:100-131) over D-dimensional rows: labels n uint64, sums k x D doubles and
 * counts k uint64 over the rows with D finite components, each when non-NULL. */
int cb_kmeans_assign_vectors(cb_context* ctx, const cb_vectors* vectors, const float* centroids, size_t k,
                             uint64_t* labels, double* sums, uint64_t* counts);

/* ---- RANSAC ----------------------------------------------------------------------------------
 * Replaces TransformRANSACEstimator<RigidTransform3f>::computeResiduals + the inlier scan of
 * RandomSampleConsensusBase::estimate (model_estimation/ransac_transform_estimator.hpp:90-98,
 * model_estimation/ransac_base.hpp:96-101): inlier COUNTS of H hypotheses over n pairs.
 * dst/src are paired clouds of equal size (pair i = point with original index i in both). */
int cb_ransac_score(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src, const float* T_h, size_t H,
                    float thresh, uint32_t* counts);
/* Residuals of one model (computeResiduals) into out[n], and inlier indices (<= thresh). */
int cb_ransac_residuals(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src, const float* T12,
                        float thresh, float* residuals, uint64_t* inliers, size_t* num_inliers);
typedef struct cb_ransac_result {
  float T[12];
  uint64_t iterations;
  uint64_t num_inliers;
  uint64_t best_iteration;
  double gpu_ms_total;
  uint64_t kernel_launches;
} cb_ransac_result;
/* RandomSampleConsensusBase::estimate() for rigid transforms (ransac_base.hpp:64-131) with the seed
 * injected in place of std::random_device (:73). Hypotheses are generated on the host in the
 * reference's order, scored on the device in batches, and scanned in order so that the kept model,
 * the early exit (:114) and the iteration count are those of the sequential loop. */
int cb_ransac_rigid(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src, uint32_t seed,
                    size_t inlier_count_thresh, size_t max_iter, float thresh, int re_estimate,
                    cb_ransac_result* res, uint64_t* inliers, float* residuals);

/* ---- plane RANSAC -----------------------------------------------------------------------------
 * Planes are float32[4] (n0, n1, n2, d): the coefficients of Eigen::Hyperplane<float, 3>. The residual of point p is
 * HyperplaneRANSACEstimator::computeResiduals' absDistance (model_estimation/ransac_hyperplane_estimator.hpp:47-55),
 * r = |((n0 x) + ((n1 y) + (n2 z))) + d| in fp32, and p is an inlier iff r <= thresh (ransac_base.hpp:96-101): NaN
 * residuals never are, and a negative or NaN threshold admits nothing. Single GPU: a cloud with index_offset != 0
 * gives CB_ERR_UNSUPPORTED.
 * cb_plane_score: the inlier counts of H planes (planes4 = H x 4 floats) over the cloud, one pass per batch of
 * planes; replaces computeResiduals + the scan for each hypothesis. */
int cb_plane_score(cb_context* ctx, const cb_cloud* cloud, const float* planes4, size_t H, float thresh,
                   uint32_t* counts);
/* computeResiduals(plane) (:47-55) into residuals[n] and the inlier scan (ransac_base.hpp:96-101): inliers ascending,
 * *num_inliers of them. residuals and inliers may be NULL. */
int cb_plane_residuals(cb_context* ctx, const cb_cloud* cloud, const float* plane4, float thresh, float* residuals,
                       uint64_t* inliers, size_t* num_inliers);
typedef struct cb_ransac_plane_result {
  float plane[4];            /* the model: re-estimated when re_estimate != 0, else the kept hypothesis */
  float hyp_plane[4];        /* the kept hypothesis before re-estimation (NaN when none was kept) */
  uint64_t iterations;       /* getNumberOfPerformedIterations() */
  uint64_t best_iteration;   /* 0-based iteration of the kept hypothesis */
  uint64_t num_inliers;
  double gpu_ms_total;       /* device time of the call */
  double gpu_ms_fit;         /* ... of which the hypothesis fits */
  double gpu_ms_score;       /* ... the scoring of the hypotheses */
  double gpu_ms_reestimate;  /* ... the masked moments of the re-estimation */
  double gpu_ms_final;       /* ... the final residuals and the inlier compaction */
  uint64_t kernel_launches;
} cb_ransac_plane_result;
/* RandomSampleConsensusBase::estimate() (ransac_base.hpp:64-131) with HyperplaneRANSACEstimator<float, 3>
 * (PlaneRANSACEstimator3f), sample size 3, the seed injected in place of std::random_device (:73); DESIGN §4.12.
 * Samples are drawn on the host in the reference's order, fitted on the device by the closed form of the 3-point
 * plane, scored in batches of growing size, and scanned in order, so that the kept hypothesis, the early exit (:114)
 * and the iteration count are those of the sequential loop. Re-estimation (:118-128): PCA of the kept hypothesis's
 * inliers, moments summed in double on the device. No hypothesis with sample_size inliers: NaN plane, 0 inliers.
 * inliers (n entries) and residuals (n) may be NULL. A context with a communicator of more than one rank:
 * CB_ERR_UNSUPPORTED. */
int cb_ransac_plane(cb_context* ctx, const cb_cloud* cloud, uint32_t seed, size_t inlier_count_thresh,
                    size_t max_iter, float thresh, int re_estimate, cb_ransac_plane_result* res, uint64_t* inliers,
                    float* residuals);

/* ---- non-rigid ICP: dense rigid warp field ------------------------------------------------------
 * cb_warp_icp_* replaces SimpleCombinedMetricDenseRigidWarpFieldICP3f (registration/icp_common_instances.hpp:99-144,
 * 284-285) = CombinedMetricDenseWarpFieldICP (registration/icp_warp_field_combined_metric_dense.hpp) on the loop of
 * IterativeClosestPointBase::estimate (icp_base.hpp:68-87); DESIGN §4.13. Every source point i carries its own rigid
 * transform T_i (float32[12] per point, row-major [R | t]). One ICP iteration: the 1-NN of T_i s_i in the destination
 * within max_d2 (the grid search of cb_find_correspondences), then estimateDenseWarpFieldCombinedMetric
 * (warp_field_estimation.hpp:368-715): per point 6 unknowns (Euler a, b, c and a translation) linearised about zero,
 * point-to-point (3 rows, weight sqrt(w_pt)) and point-to-plane (1 row, sqrt(w_pl)) data terms, and per regularisation
 * arc 6 Huber-loss rows of weight sqrt(stiffness) sqrt(exp(reg_coeff d2)); Gauss-Newton steps solved by a Jacobi-
 * preconditioned conjugate gradient with zero initial guess; then T_i <- rotation(dT_i T_i) (TransformSet::preApply)
 * and last_delta = sqrt(max_i |dR_i - I|_F^2 + |dt_i|^2). The loop stops when last_delta < tol or at max_iter.
 * Regularisation neighbourhoods: a host CSR in the layout cb_radius_search returns (n_reg lists; list j is entries
 * offsets[j] .. offsets[j+1]-1 of index / value). Each list N gives the arcs (N[0], N[j]) for j >= 1 with value
 * N[j].value; an empty list gives none (the reference's size() - 1 underflows there), and a self-arc (N[0] == N[j])
 * gives none (its two Jacobian entries cancel). Rejected: a neighbour index outside [0, n_src) (CB_ERR_INVALID),
 * w_pl > 0 on a destination without normals (CB_ERR_INVALID; the reference returns identities and later reads the
 * missing normals), any non-default correspondence-engine option, a cloud with index_offset != 0, a context with
 * more than one rank, and clouds of 2^31 - 1 points or more (CB_ERR_UNSUPPORTED; point indices travel as signed
 * 32-bit values through the search). A non-finite source point gets no
 * correspondence. With no data term (both weights <= 0, or no correspondence) every T_i of the iteration is the
 * identity and the estimator reports false (:398-408). */
typedef struct cb_warp_params {
  float w_pt;            /* point_to_point_weight_, default 0 */
  float w_pl;            /* point_to_plane_weight_, default 1 */
  float stiffness;       /* stiffness_weight_, default 1 */
  float huber;           /* huber_boundary_, default 1e-4 */
  float gn_tol;          /* gauss_newton_convergence_tol_, default 1e-5 */
  float cg_tol;          /* conjugate_gradient_convergence_tol_, default 1e-5 */
  float tol;             /* icp_base.hpp:25, default 1e-5 */
  float max_d2;          /* SQUARED; correspondence_search_kd_tree.hpp:49, default 0.01*0.01 */
  float reg_coeff;       /* RBFKernelWeightEvaluator<float, float, true>: -0.5f / (sigma * sigma); default sigma 1 */
  int32_t max_iter;      /* icp_base.hpp:24, default 15 */
  uint64_t max_gn_iter;  /* default 10 */
  uint64_t max_cg_iter;  /* default 1000 */
  /* correspondence-engine options as in cb_icp_params; only the defaults are supported here */
  int32_t search_dir;
  int32_t require_reciprocal;
  int32_t one_to_one;
  int32_t reserved_;
  double inlier_fraction;
} cb_warp_params;

typedef struct cb_warp_result {
  int32_t iterations;       /* getNumberOfPerformedIterations() */
  int32_t converged;        /* hasConverged(): last_delta < tol */
  float last_delta;
  int32_t reserved_;
  uint64_t num_corr;        /* correspondences of the last iteration */
  uint64_t gn_steps;        /* Gauss-Newton steps over all iterations */
  uint64_t cg_iterations;   /* conjugate-gradient iterations over all steps */
  double gpu_ms_search;     /* CUDA-event time of the correspondence searches */
  double gpu_ms_solve;      /* ... of the assembly, CG and compose kernels */
  uint64_t kernel_launches;
} cb_warp_result;

typedef struct cb_warp_solve_result {
  int32_t converged;        /* the estimator's return value */
  float cg_error;           /* sqrt(|r|^2 / |b|^2) after the last step's CG (0 when |b| = 0) */
  uint64_t gn_steps;
  uint64_t cg_iterations;   /* over all steps */
  uint64_t cg_iterations_last;
  uint64_t kernel_launches;
} cb_warp_solve_result;

typedef struct cb_warp_icp cb_warp_icp;

void cb_warp_default_params(cb_warp_params* p);
/* dst (with normals for w_pl > 0) and src must outlive the object. The neighbourhoods are validated, uploaded once and
 * turned into a per-point arc incidence on the device (stable radix sort by point). */
int cb_warp_icp_create(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src, const uint64_t* reg_offsets,
                       const int64_t* reg_index, const float* reg_value, size_t n_reg, cb_warp_icp** out);
void cb_warp_icp_destroy(cb_warp_icp* icp);
/* estimate() followed by getTransform(): T_init (n_src x 12, NULL = identities) -> T_out (n_src x 12). */
int cb_warp_icp_estimate(cb_warp_icp* icp, const cb_warp_params* prm, const float* T_init, float* T_out,
                         cb_warp_result* res);
/* estimateDenseWarpFieldCombinedMetric on the source transformed by T_src (n_src x 12, NULL = identities) with the
 * caller's correspondences (dst index corr_first[c], src index corr_second[c]; corr_value may be NULL: the Simple
 * instance weighs data terms with UnityWeightEvaluator). T_out (n_src x 12) = the estimated per-point transforms;
 * x_out (n_src x 6, may be NULL) = the estimator's unknowns (a, b, c, tx, ty, tz) per point, from which T_out is
 * built (with one Gauss-Newton step: the CG solution of the normal equations). An index out of range: CB_ERR_INVALID. */
int cb_warp_icp_solve(cb_warp_icp* icp, const cb_warp_params* prm, const float* T_src, const uint64_t* corr_first,
                      const uint64_t* corr_second, const float* corr_value, size_t n_corr, float* T_out, float* x_out,
                      cb_warp_solve_result* res);
/* computeResiduals() (icp_warp_field_combined_metric_dense.hpp:216-236) for the per-point transforms T (n_src x 12):
 * unbounded 1-NN of T_i s_i, out[i] = w_pt |d - p|^2 + w_pl (n_d . (d - p))^2; NaN when dst is empty. */
int cb_warp_icp_residuals(cb_warp_icp* icp, const cb_warp_params* prm, const float* T, float* out);
/* getCorrespondences() after the last iteration of the last estimate(), ascending source index; arrays hold n_src. */
int cb_warp_icp_correspondences(cb_warp_icp* icp, uint64_t* index_first, uint64_t* index_second, float* value,
                                size_t* count);
/* Projective correspondence search for the dense warp field: SimpleCombinedMetricDenseRigidWarpFieldProjectiveICP3f
 * (registration/icp_common_instances.hpp:233-245, 298-299), whose updateCorrespondences() calls the projective engine's
 * findCorrespondences(transform_) (correspondence_search/correspondence_search_projective.hpp:68-75, 156-209). K9, w, h
 * and E12 as in cb_icp_set_projection, whose index map this call builds over the destination cloud and keeps on the
 * device until the next call or cb_warp_icp_destroy. From then on cb_warp_icp_estimate matches every warped point
 * T_i s_i to the destination point its pixel shows, kept iff its squared distance is < max_d2: the contract of
 * DESIGN §4.21 on the warped points (DESIGN §4.22). cb_warp_icp_residuals stays the kd-tree search, as the reference's
 * computeResiduals. K9 = NULL detaches the projection and restores the grid search. w or h = 0: no correspondences (the
 * estimate returns identities with last_delta = 0). Non-finite K9 or E12, w h >= 2^32: CB_ERR_INVALID. On an error
 * the projection attached before the call (or none) stays in force; a successful call makes cb_warp_icp_correspondences
 * return CB_ERR_INVALID until the next estimate. Launches: 3 (2 for an empty destination cloud). */
int cb_warp_icp_set_projection(cb_warp_icp* icp, const float* K9, size_t w, size_t h, const float* E12);

/* ---- non-rigid ICP: sparse rigid warp field on control nodes ------------------------------------
 * cb_sparse_warp_icp_* replaces SimpleCombinedMetricSparseRigidWarpFieldICP3f (registration/icp_common_instances.hpp:
 * 146-199, 313-314) = CombinedMetricSparseWarpFieldICP (registration/icp_warp_field_combined_metric_sparse.hpp) on the
 * loop of IterativeClosestPointBase::estimate (icp_base.hpp:68-87); DESIGN §4.14. n_ctrl control nodes carry one rigid
 * transform each (float32[12], row-major [R | t]); source point i carries a control list (the nodes n_ik that move it,
 * with squared distances d2_ik) and its dense transform is resampleTransforms (warp_field_utilities.hpp:14-48):
 * w_ik = exp(ctrl_coeff d2_ik) over the list in the given order, T_i = (rotation(sum w R / W), sum w t / W),
 * W = sum w, the identity when W = 0. One ICP iteration: the 1-NN of T_i s_i within max_d2 (as cb_warp_icp), then
 * estimateSparseWarpFieldCombinedMetric (warp_field_estimation.hpp:1388-1846): 6 unknowns per node starting at zero,
 * point i linearised at the weighted mean (sum_k w_ik x_{n_ik}) / W_i of its list sorted by node, the dense
 * estimator's data rows with the entry of node n_ik scaled by sqrt(w) w_ik / W_i and the residual by sqrt(w) (rows
 * of zero when W_i = 0), and the Huber arcs (N[0], N[j]) of the node neighbourhoods as in cb_warp_icp; then the node
 * transforms are composed as TransformSet::preApply, resampled onto the points, and
 * last_delta = sqrt(max_j |dR_j - I|_F^2 + |dt_j|^2) over the nodes.
 * Defined here where the reference is undefined or silent: a control-list count other than n_src, a control index
 * >= n_ctrl and a regularisation index >= n_ctrl are CB_ERR_INVALID; an empty control list gives the identity and
 * no data rows; a node no point and no arc touches keeps the identity; duplicate nodes in one list are summed (the
 * sort is stable). Everything else (empty neighbourhoods, self-arcs, non-finite points, w_pl > 0 without normals,
 * engine options, ranks, the 2^31 - 1 point limit) follows cb_warp_icp. */
typedef struct cb_sparse_warp_params {
  cb_warp_params base;   /* the dense parameters; base.reg_coeff weighs the regularisation arcs */
  float ctrl_coeff;      /* control weights, RBFKernelWeightEvaluator<float, float, true>: -0.5f / sigma^2, sigma 1 */
  int32_t reserved_;
} cb_sparse_warp_params;

typedef struct cb_sparse_warp_result {
  int32_t iterations;       /* getNumberOfPerformedIterations() */
  int32_t converged;        /* hasConverged(): last_delta < tol */
  float last_delta;
  int32_t reserved_;
  uint64_t num_corr;        /* correspondences of the last iteration */
  uint64_t gn_steps;        /* Gauss-Newton steps over all iterations */
  uint64_t cg_iterations;   /* conjugate-gradient iterations over all steps */
  double gpu_ms_search;     /* CUDA-event time of the correspondence searches */
  double gpu_ms_resample;   /* ... of resampling node transforms onto the points (after each compose) */
  double gpu_ms_assemble;   /* ... of the per-point and per-node assembly */
  double gpu_ms_cg;         /* ... of the CG launches */
  uint64_t kernel_launches;
} cb_sparse_warp_result;

typedef struct cb_sparse_warp_icp cb_sparse_warp_icp;

void cb_sparse_warp_default_params(cb_sparse_warp_params* p);
/* dst (with normals for w_pl > 0) and src must outlive the object. Control lists: a host CSR of n_ctrl_lists lists
 * (= n_src) of (node index, squared distance), e.g. the kNN of each source point among the nodes; regularisation
 * neighbourhoods: a CSR over the nodes as in cb_warp_icp_create. Both are validated and uploaded once; the
 * node -> (point, entry) and arc incidences are built on the device by the stable radix sort. */
int cb_sparse_warp_icp_create(cb_context* ctx, const cb_cloud* dst, const cb_cloud* src, const uint64_t* ctrl_offsets,
                              const int64_t* ctrl_index, const float* ctrl_value, size_t n_ctrl_lists, size_t n_ctrl,
                              const uint64_t* reg_offsets, const int64_t* reg_index, const float* reg_value,
                              size_t n_reg, cb_sparse_warp_icp** out);
void cb_sparse_warp_icp_destroy(cb_sparse_warp_icp* icp);
/* estimate() followed by getTransform() and getDenseWarpField(): T_init (n_ctrl x 12, NULL = identities) -> T_out
 * (n_ctrl x 12); T_dense_out (n_src x 12, may be NULL) = the resampled per-point transforms. */
int cb_sparse_warp_icp_estimate(cb_sparse_warp_icp* icp, const cb_sparse_warp_params* prm, const float* T_init,
                                float* T_out, float* T_dense_out, cb_sparse_warp_result* res);
/* estimateSparseWarpFieldCombinedMetric on the source transformed by T_dense_src (n_src x 12, NULL = identities) with
 * the caller's correspondences (as cb_warp_icp_solve). T_out (n_ctrl x 12) = the estimated node transforms; x_out
 * (n_ctrl x 6, may be NULL) = the unknowns (a, b, c, tx, ty, tz) per node. An index out of range: CB_ERR_INVALID. */
int cb_sparse_warp_icp_solve(cb_sparse_warp_icp* icp, const cb_sparse_warp_params* prm, const float* T_dense_src,
                             const uint64_t* corr_first, const uint64_t* corr_second, const float* corr_value,
                             size_t n_corr, float* T_out, float* x_out, cb_warp_solve_result* res);
/* resampleTransforms (warp_field_utilities.hpp:14-48) with the control weights of prm: node transforms T_ctrl
 * (n_ctrl x 12) -> T_dense_out (n_src x 12). */
int cb_sparse_warp_icp_resample(cb_sparse_warp_icp* icp, const cb_sparse_warp_params* prm, const float* T_ctrl,
                                float* T_dense_out);
/* computeResiduals() (icp_warp_field_combined_metric_sparse.hpp:243-263) for the dense field T_dense (n_src x 12), as
 * cb_warp_icp_residuals. */
int cb_sparse_warp_icp_residuals(cb_sparse_warp_icp* icp, const cb_sparse_warp_params* prm, const float* T_dense,
                                 float* out);
/* getCorrespondences() after the last iteration of the last estimate(), ascending source index; arrays hold n_src. */
int cb_sparse_warp_icp_correspondences(cb_sparse_warp_icp* icp, uint64_t* index_first, uint64_t* index_second,
                                       float* value, size_t* count);
/* Projective correspondence search for the sparse warp field: SimpleCombinedMetricSparseRigidWarpFieldProjectiveICP3f
 * (registration/icp_common_instances.hpp:233-245, 327-328), whose updateCorrespondences() calls the projective engine's
 * findCorrespondences(transform_dense_) (icp_warp_field_combined_metric_sparse.hpp:208-209). The rules of
 * cb_warp_icp_set_projection, on the points warped by the resampled dense field. */
int cb_sparse_warp_icp_set_projection(cb_sparse_warp_icp* icp, const float* K9, size_t w, size_t h, const float* E12);

/* ---- covariance / PCA ------------------------------------------------------------------------
 * Replaces Covariance<float,3>::operator() (core/covariance.hpp:31-80) and
 * PrincipalComponentAnalysis<float,3> (core/principal_component_analysis.hpp:76-84).
 * cov / evecs row-major 3x3, eigenvalues descending, evecs right-handed. Returns 1 if n >= 2,
 * else fills NaN and returns 0 (covariance.hpp:35-38). */
int cb_mean_cov(cb_context* ctx, const cb_cloud* pts, float* mean3, float* cov9);
int cb_pca(cb_context* ctx, const cb_cloud* pts, float* mean3, float* cov9, float* evals3, float* evecs9);

/* ---- covariance / PCA over D-dimensional vector sets -------------------------------------------
 * Covariance<float, D>::operator()(points, mean, cov) and its subset / iterator overloads (core/covariance.hpp:30-179)
 * for any D: subset NULL = every row, else the m listed rows (duplicates count twice; an index >= n is
 * CB_ERR_INVALID). mean D floats, cov D x D row-major. fp64 accumulation about a pivot (DESIGN §4.18); at D = 3 the
 * bits of cb_mean_cov. A non-finite value in dimension j makes row and column j of cov NaN. Fewer than
 * min_sample_size rows: NaN mean and cov, returns 0. Otherwise returns 1; n = 1 gives mean = the row and a NaN cov,
 * n = 0 a NaN mean and cov = -0 (whole set) or +0 (subset), the reference's expressions. One GPU: a context with
 * several ranks returns CB_ERR_UNSUPPORTED. */
int cb_vectors_mean_cov(cb_context* ctx, const cb_vectors* v, const uint64_t* subset, size_t m,
                        size_t min_sample_size, float* mean, float* cov);
/* PrincipalComponentAnalysis<float, D> constructors (core/principal_component_analysis.hpp:17-31,76-84): the above,
 * then the eigen-decomposition of the fp32 covariance (cb_solve_sym_eigen; at D = 3 cb_pca's). evals D descending,
 * evecs D x D row-major with the eigenvectors as columns. Returns as cb_vectors_mean_cov (0: all NaN). */
int cb_vectors_pca(cb_context* ctx, const cb_vectors* v, const uint64_t* subset, size_t m, size_t min_sample_size,
                   float* mean, float* cov, float* evals, float* evecs);
/* PrincipalComponentAnalysis::project(points, k) / project<k> (principal_component_analysis.hpp:46-57) with
 * cb_vectors_pca's mean and evecs (first k columns), 1 <= k <= D: out_j = fold over d = 0 .. D-1 of
 * acc = acc + E[d][j] * (p_d - mean_d) from acc = 0, fp32 without FMA. n x k rows to out_host and / or a new vector
 * set *out_device (either may be NULL, not both). */
int cb_vectors_project(cb_context* ctx, const cb_vectors* v, const float* mean, const float* evecs, int k,
                       float* out_host, cb_vectors** out_device);
/* reconstruct(points) / reconstruct<k> (principal_component_analysis.hpp:59-68) of q (n x k, 1 <= k <= D) into D
 * dimensions: out_r = (fold over j = 0 .. k-1 of acc = acc + E[r][j] * q_j from acc = 0) + mean_r, fp32 without FMA. */
int cb_vectors_reconstruct(cb_context* ctx, const cb_vectors* q, const float* mean, const float* evecs, int D,
                           float* out_host, cb_vectors** out_device);

/* ---- multidimensional scaling ------------------------------------------------------------------
 * computeDistancePreservingSpectralEmbedding / MultidimensionalScaling<float, D>
 * (utilities/multidimensional_scaling.hpp:35-83, 86-121) on an n x n fp32 distance matrix held as a cb_vectors with
 * D = n (row i = row i of the matrix). Entries are squared once in fp32 unless distances_are_squared. B is the symmetric
 * matrix whose entries for i >= j are -1/2 (E_ij - r_i - c_j + g) (row means r, column means c, grand mean g, fp64): the
 * lower triangle of -1/2 J E J, the triangle the reference's eigen-solver reads. nev = estimate_dim ?
 * min(max_dim + 1, n - 1) : max_dim eigenpairs of largest |lambda| (descending |lambda|, the positive value first at
 * equal magnitude) are found with fp64 products on the device; then negative eigenvalues are clamped to 0, the dimension
 * is max_dim or, with estimate_dim, estimateEmbeddingDimensionEigengap (:9-31) of the clamped values, and each
 * eigenvector is signed so that its largest-magnitude component is positive (lowest index on ties).
 * eigenvalues: nev floats (*nev is set); *dim is set; the embedding diag(sqrt(lambda)) V^T, dim x n in the reference, is
 * written as n x dim rows to embedded_host (n x max_dim floats of room) and / or a new vector set *embedded_device
 * (either may be NULL). nev outside [1, n - 1], estimate_dim with max_dim >= n, or a non-square set (D != n) is
 * CB_ERR_INVALID; a context with several ranks is CB_ERR_UNSUPPORTED. A non-finite (squared) entry returns 0 with NaN
 * outputs (dim as without estimation); no convergence within the restart cap returns CB_ERR_UNSUPPORTED. Returns 1. */
int cb_vectors_mds(cb_context* ctx, const cb_vectors* dist, size_t max_dim, int estimate_dim, int distances_are_squared,
                   float* eigenvalues, size_t* nev, size_t* dim, float* embedded_host, cb_vectors** embedded_device);

/* ---- depth images <-> clouds -------------------------------------------------------------------------------------
 * core/image_point_cloud_conversions.hpp with MetricDepth = float, under the contract of DESIGN §4.20. A converter is
 * DepthValueConverter<RawDepth, float>(scale) (:7-24) or, truncated, TruncatedDepthValueConverter(scale, max_depth)
 * (:26-51): metric = (1.0f / scale) * float(raw), truncated to 0 at or above max_depth. scale must be finite and
 * nonzero. Intrinsics K are float32[9], row-major, any invertible 3 x 3; extrinsics are float32[12] [R | t] taken as a
 * rigid transform, or NULL. Images are row-major, pixel k = y * w + x; rgb is 3 bytes per pixel. w * h >= 2^32 pixels
 * or n >= 2^32 points is CB_ERR_UNSUPPORTED. One GPU. */
typedef enum cb_raw_depth { CB_DEPTH_U16 = 0 /* unsigned short */, CB_DEPTH_F32 = 1 /* float */ } cb_raw_depth;
typedef struct cb_depth_converter {
  int32_t raw_type;  /* cb_raw_depth */
  int32_t truncated; /* 0: DepthValueConverter, 1: TruncatedDepthValueConverter */
  float scale;       /* the converters' mult */
  float max_depth;   /* truncated only */
} cb_depth_converter;

/* depthImageToPoints (:53-147), depthImageToPointsNormals (:149-344), RGBDImagesToPointsColors (:346-473) and
 * RGBDImagesToPointsNormalsColors (:475-695), each with and without extrinsics, and PointCloud's image constructors /
 * fromDepthImage / fromRGBDImages (utilities/point_cloud.hpp:83-116, 463-500). depth (w * h raw values) and rgb (NULL,
 * or 3 w h bytes) may each be host memory or device memory of the context's device (another device's memory is
 * CB_ERR_INVALID). A device image is read on the context's stream without waiting for any other stream: the work that
 * wrote it must have completed (e.g. its stream synchronised) before the call. want_normals selects the ...Normals variants. keep_invalid: all
 * w * h pixels in pixel order (invalid ones as computed, normals NaN where there is none); else the kept pixels in
 * ascending pixel order: p.z > 0, or with normals a non-NaN normal. *count is set. points / normals / colors (each may
 * be NULL; colors needs rgb, normals needs want_normals) are host arrays with room for 3 w h floats;
 * *out_device (NULL = none) receives a new cloud of the points (and normals) that cb_cloud_grid_downsample,
 * cb_cloud_estimate_normals and cb_icp_create take. Launches per call: 1 with keep_invalid, else 5. */
int cb_depth_image_to_points(cb_context* ctx, const void* depth, const unsigned char* rgb, size_t w, size_t h,
                             const cb_depth_converter* conv, const float* K, const float* extrinsics, int want_normals,
                             int keep_invalid, float* points, float* normals, float* colors, size_t* count,
                             cb_cloud** out_device);

/* pointsToDepthImage (:697-772) and, with colors, pointsColorsToRGBDImages (:774-863), with and without extrinsics.
 * The points are n packed xyz on the host (xyz) or a cloud (cloud, n ignored); exactly one of them. colors: NULL or
 * 3 n host floats, given together with rgb. Writes w * h raw values to depth (host) and 3 w h bytes to rgb (host). Per
 * pixel the smallest raw depth wins, the lowest point index on ties, and the colour is the winner's; a raw depth that
 * does not fit an unsigned short is skipped, a colour byte saturates (NaN -> 0). Launches per call: 2. */
int cb_points_to_depth_image(cb_context* ctx, const float* xyz, const cb_cloud* cloud, size_t n, const float* colors,
                             const float* K, const float* extrinsics, const cb_depth_converter* conv, size_t w,
                             size_t h, void* depth, unsigned char* rgb);

/* pointsToIndexMap (:865-934), with and without extrinsics, IndexT = uint64_t: per pixel the index of the point of
 * smallest camera-frame z, the lowest index on ties, plus the cloud's index_offset when the points are a cloud;
 * UINT64_MAX where no point projects. Points as in
 * cb_points_to_depth_image. Launches per call: 2. */
int cb_points_to_index_map(cb_context* ctx, const float* xyz, const cb_cloud* cloud, size_t n, const float* K,
                           const float* extrinsics, size_t w, size_t h, uint64_t* index_map);

/* transformPoints(tform, in, out) — core/space_transformations.hpp:203-216 (host in, host out). */
int cb_transform_points(cb_context* ctx, const float* T12, const float* xyz, size_t n, float* out);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* CILANTRO_B200_H_ */
