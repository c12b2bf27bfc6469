// The sample sequence of RandomSampleConsensusBase::estimate (model_estimation/ransac_base.hpp:72-91): a partial
// Fisher-Yates shuffle of a permutation that persists across iterations, driven by std::mt19937 with the seed
// injected in place of std::random_device (:73). Shared by the rigid (ransac.cu) and plane (ransac_plane.cu)
// estimators.
#pragma once
#include <cstddef>
#include <cstdint>
#include <random>
#include <utility>
#include <vector>

namespace cb {

class RansacSampler {
public:
  RansacSampler(size_t n, uint32_t seed) : perm_(n), rng_(seed) {
    for (size_t i = 0; i < n; i++) perm_[i] = i;
  }
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

}  // namespace cb
