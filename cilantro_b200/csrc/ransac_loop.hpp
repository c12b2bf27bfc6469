// The hypothesis loop of RandomSampleConsensusBase::estimate (model_estimation/ransac_base.hpp:64-114), shared by the
// rigid (ransac.cu) and plane (ransac_plane.cu) estimators. The samples are drawn on the host in the reference's
// order, a batch of them is fitted and scored by the model, and the batch's counts are scanned in order, so that the
// kept hypothesis, the early exit (:114) and the iteration count are those of the sequential loop. Host code only:
// tests/cpp/test_ransac_loop.cpp compiles it with g++ and drives it with a fake model.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <random>
#include <utility>
#include <vector>

namespace cb {

// The sample sequence (:72-91): a partial Fisher-Yates shuffle of a permutation that persists across iterations,
// driven by std::mt19937 with the seed injected in place of std::random_device (:73).
class RansacSampler {
public:
  RansacSampler(size_t n, uint32_t seed) : perm_(n), rng_(seed) {
    for (size_t i = 0; i < n; i++) perm_[i] = i;
  }
  size_t size() const { return perm_.size(); }
  // the next sample (:83-91): sample_size <= n indices into out
  void next(size_t sample_size, uint32_t* out) {
    size_t prev_size = perm_.size();
    for (size_t i = 0; i < sample_size; i++) {
      std::uniform_int_distribution<size_t> dist(0, prev_size - 1);
      const size_t r = dist(rng_);
      out[i] = (uint32_t)perm_[r];
      prev_size--;
      std::swap(perm_[r], perm_[prev_size]);
    }
  }

private:
  std::vector<size_t> perm_;
  std::mt19937 rng_;
};

// Both models' minimum sample: 3 point pairs of a rigid transform, 3 points of a plane. Samples are stored with this
// stride whatever the clamped sample size.
constexpr size_t kRansacSample = 3;

struct RansacRun {
  size_t sample_size = 0;  // kRansacSample clamped to n (:67)
  size_t target = 0;       // the target inlier count clamped to n (:68)
  size_t iterations = 0;
  size_t best_iteration = 0;  // 0-based iteration of the kept hypothesis
  size_t best_count = 0;
  bool have_best = false;  // a hypothesis reached sample_size inliers
};

// Runs the loop over the sampler's n data points. The caller builds the sampler (8 bytes per point, filled on the
// host) before it starts the clock of its gpu_ms_total, which times the loop and not that set-up. Batches hold
// first_batch hypotheses, doubling per batch up to max_batch (an early exit wastes at most as many hypotheses as
// already ran). The model's hooks, each returning 0 or an error code that ends the loop and is returned:
//   fit(const uint32_t* idx, size_t nb, size_t sample_size): fit the nb samples idx[3 b .. 3 b + sample_size);
//   score(size_t nb, uint32_t* counts): the inlier count of each of the nb hypotheses into counts;
//   keep(size_t b): hypothesis b of the batch becomes the best one (void).
template <class Model>
int ransac_loop(RansacSampler& sampler, size_t target, size_t max_iter, size_t first_batch, size_t max_batch,
                Model& model, RansacRun* run) {
  RansacRun& r = *run;
  r = RansacRun();
  r.sample_size = std::min(kRansacSample, sampler.size());  // :67
  r.target = std::min(target, sampler.size());               // :68
  std::vector<uint32_t> idx(kRansacSample * max_batch, 0u), counts(max_batch);
  size_t batch = first_batch;
  bool done = false;
  while (!done && r.iterations < max_iter) {
    const size_t nb = std::min(batch, max_iter - r.iterations);
    batch = std::min(2 * batch, max_batch);
    for (size_t b = 0; b < nb; b++) sampler.next(r.sample_size, &idx[kRansacSample * b]);
    if (int e = model.fit(idx.data(), nb, r.sample_size)) return e;  // :94
    if (int e = model.score(nb, counts.data())) return e;            // :95-101
    for (size_t b = 0; b < nb && !done; b++) {
      r.iterations++;
      const size_t cnt = counts[b];
      if (cnt < r.sample_size) continue;  // :104
      if (cnt > r.best_count) {           // :107 (model_inliers_ starts empty)
        r.best_count = cnt;
        r.best_iteration = r.iterations - 1;
        r.have_best = true;
        model.keep(b);
      }
      done = r.best_count >= r.target;  // :114
    }
  }
  return 0;
}

}  // namespace cb
