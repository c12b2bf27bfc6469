// Same include path as cilantro's clustering/mean_shift.hpp: MeanShift3f over cb_cloud_mean_shift. The kernel
// evaluator maps by kind (UnityWeightEvaluator, RBFKernelWeightEvaluator<float, float, true>); any other evaluator type
// is a compile-time error. Semantics and tie rule: include/cilantro_b200.h (cb_cloud_mean_shift), DESIGN §4.11.
#pragma once
#include <limits>
#include <vector>

#include "../b200_shims.hpp"
#include "../core/common_pair_evaluators.hpp"

namespace cilantro {

// clustering/mean_shift.hpp:9-140 for float and 3 dimensions; the ClusteringBase maps are indexed by seed
template <typename PointIndexT = size_t, typename ClusterIndexT = size_t>
class MeanShift3f {
public:
  using Scalar = float;
  enum { Dimension = 3 };
  using SearchTree = KDTree3f<PointIndexT>;
  using ClusterToPointIndicesMap = std::vector<std::vector<PointIndexT>>;
  using PointToClusterIndexMap = std::vector<ClusterIndexT>;

  MeanShift3f(const ConstVectorSetMatrixMap3f& points, size_t /*max_leaf_size*/ = 10)
      : n_(points.cols()), own_(points), cloud_(own_.h) {}
  // reuses the tree's device-resident cloud (no second upload or index build)
  MeanShift3f(const SearchTree& kd_tree) : n_(kd_tree.getPointsMatrixMap().cols()), cloud_(kd_tree.b200_cloud()) {}

  // :37-115
  template <class KernelEvaluatorT = UnityWeightEvaluator<float, float>>
  MeanShift3f& cluster(const ConstVectorSetMatrixMap3f& seeds, float kernel_radius, size_t max_iter, float cluster_tol,
                       float convergence_tol = std::numeric_limits<float>::epsilon(),
                       const KernelEvaluatorT& evaluator = KernelEvaluatorT()) {
    run(seeds.data(), seeds.cols(), kernel_radius, max_iter, cluster_tol, convergence_tol, evaluator);
    return *this;
  }
  // :118-124: every point is a seed (the points already on the device)
  template <class KernelEvaluatorT = UnityWeightEvaluator<float, float>>
  MeanShift3f& cluster(float kernel_radius, size_t max_iter, float cluster_tol,
                       float convergence_tol = std::numeric_limits<float>::epsilon(),
                       const KernelEvaluatorT& evaluator = KernelEvaluatorT()) {
    run(nullptr, n_, kernel_radius, max_iter, cluster_tol, convergence_tol, evaluator);
    return *this;
  }

  const VectorSet3f& getShiftedSeeds() const { return shifted_; }
  const VectorSet3f& getClusterModes() const { return modes_; }
  size_t getNumberOfPerformedIterations() const { return iterations_; }
  // ClusteringBase getters (clustering/clustering_base.hpp)
  const ClusterToPointIndicesMap& getClusterToPointIndicesMap() const { return clusters_; }
  const PointToClusterIndexMap& getPointToClusterIndexMap() const { return p2c_; }
  size_t getNumberOfClusters() const { return clusters_.size(); }
  size_t getNumberOfPoints() const { return p2c_.size(); }

private:
  template <class KernelEvaluatorT>
  void run(const float* seeds, size_t ns, float kernel_radius, size_t max_iter, float cluster_tol, float convergence_tol,
           const KernelEvaluatorT& evaluator) {
    cb_mean_shift_params p{};
    p.kernel_radius = kernel_radius;
    p.max_iter = max_iter;
    p.cluster_tol = cluster_tol;
    p.convergence_tol = convergence_tol;
    p.weight_kind = evaluator.b200_kind();  // no such member: the evaluator type has no device mapping
    p.weight_coeff = evaluator.b200_coeff();
    VectorSet3f shifted(3, ns), modes(3, ns);
    std::vector<uint64_t> p2c(ns > 0 ? ns : 1), off(ns + 1), pts(ns > 0 ? ns : 1);
    size_t m = 0;
    uint64_t it = 0;
    float none[3] = {0.f, 0.f, 0.f};
    b200::check(cb_cloud_mean_shift(b200::Context::get(), cloud_, &p, seeds ? (ns ? seeds : none) : nullptr, ns,
                              ns ? shifted.data() : none, p2c.data(), off.data(), pts.data(), ns ? modes.data() : none,
                              &m, &it, nullptr, nullptr),
          "cb_cloud_mean_shift");
    shifted_ = shifted;
    modes_ = VectorSet3f(3, m);
    for (size_t c = 0; c < m; c++) modes_.setCol(c, modes.col(c));
    clusters_.assign(m, {});
    for (size_t c = 0; c < m; c++) clusters_[c].assign(pts.begin() + (ptrdiff_t)off[c], pts.begin() + (ptrdiff_t)off[c + 1]);
    p2c_.assign(p2c.begin(), p2c.begin() + (ptrdiff_t)ns);
    iterations_ = (size_t)it;
  }

  size_t n_;
  b200::CloudHandle own_;
  cb_cloud* cloud_;
  size_t iterations_ = 0;
  VectorSet3f shifted_, modes_;
  ClusterToPointIndicesMap clusters_;
  PointToClusterIndexMap p2c_;
};

}  // namespace cilantro
