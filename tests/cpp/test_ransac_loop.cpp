// Host check of cilantro_b200/csrc/ransac_loop.hpp (the hypothesis loop of the rigid and plane RANSAC estimators).
// A fake model takes its inlier counts from a seeded table indexed by hypothesis; the loop must give what a direct
// restatement of RandomSampleConsensusBase::estimate (model_estimation/ransac_base.hpp:64-114) gives on the same
// table: the sample sequence, the clamped sample size and target, the iteration count, the kept hypothesis and its
// count, and the early exit. Every batch schedule must agree, and the batches must follow the schedule.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <numeric>
#include <random>
#include <utility>
#include <vector>

#include "ransac_loop.hpp"

static int failures = 0;
#define CHECK(cond, ...)                 \
  do {                                   \
    if (!(cond)) {                       \
      std::printf("FAIL: ");             \
      std::printf(__VA_ARGS__);          \
      std::printf("\n");                 \
      failures++;                        \
    }                                    \
  } while (0)

struct Expected {
  size_t sample_size = 0, target = 0, iterations = 0, best_iteration = 0, best_count = 0;
  bool have_best = false;
  std::vector<uint32_t> samples;  // sample_size indices per performed iteration
};

// ransac_base.hpp:64-114 with the seed injected (:73) and curr_inliers.size() read from the table
static Expected restated(size_t n, uint32_t seed, size_t target, size_t max_iter, const std::vector<uint32_t>& table) {
  Expected e;
  size_t sample_size = 3;
  if (n < sample_size) sample_size = n;  // :67
  if (target > n) target = n;            // :68
  std::vector<size_t> perm(n);
  std::iota(perm.begin(), perm.end(), size_t(0));
  std::mt19937 rng(seed);
  size_t best = 0;  // model_inliers_.size()
  while (e.iterations < max_iter) {
    size_t prev_size = n;
    for (size_t i = 0; i < sample_size; i++) {
      std::uniform_int_distribution<size_t> dist(0, prev_size - 1);
      const size_t r = dist(rng);
      e.samples.push_back((uint32_t)perm[r]);
      prev_size--;
      std::swap(perm[r], perm[prev_size]);
    }
    const size_t cnt = table[e.iterations];
    e.iterations++;
    if (cnt < sample_size) continue;
    if (cnt > best) {
      best = cnt;
      e.best_iteration = e.iterations - 1;
      e.have_best = true;
    }
    if (best >= target) break;
  }
  e.sample_size = sample_size;
  e.target = target;
  e.best_count = best;
  return e;
}

struct FakeModel {
  const std::vector<uint32_t>& table;
  int fail_batch = -1;  // score() of this batch returns an error
  size_t first = 0;     // hypothesis index of the current batch's first
  size_t fitted = 0;
  size_t kept = SIZE_MAX;
  std::vector<size_t> batches;
  std::vector<uint32_t> samples;
  int fit(const uint32_t* idx, size_t nb, size_t sample_size) {
    first = fitted;
    fitted += nb;
    batches.push_back(nb);
    for (size_t b = 0; b < nb; b++) {
      const uint32_t* s = idx + cb::kRansacSample * b;
      samples.insert(samples.end(), s, s + sample_size);
    }
    return 0;
  }
  int score(size_t nb, uint32_t* counts) {
    if ((int)batches.size() - 1 == fail_batch) return 7;
    for (size_t b = 0; b < nb; b++) counts[b] = table[first + b];
    return 0;
  }
  void keep(size_t b) { kept = first + b; }
};

int main() {
  const size_t schedules[4][2] = {{1, 1}, {7, 7}, {64, 1024}, {1024, 1024}};
  const size_t ns[] = {0, 1, 2, 3, 4, 10, 1000, 100000};
  const size_t iters[] = {0, 1, 2, 63, 64, 65, 1000, 2500};
  const uint32_t seeds[] = {0u, 1u, 12345u, 4294967295u};
  size_t cases = 0, exits = 0, kept = 0;
  for (size_t n : ns) {
    const size_t targets[] = {0, 1, 2, 3, n / 2 + n % 2, n, n + 1, n + 100};
    for (size_t target : targets)
      for (size_t max_iter : iters)
        for (uint32_t seed : seeds) {
          // counts under a ceiling that rises with the iteration, so that the best count improves several times
          // and the target, when reachable, is met at varied positions within and across batches
          std::mt19937 gen(seed ^ (uint32_t)(n * 7919 + target * 104729 + max_iter));
          std::vector<uint32_t> table(max_iter);
          for (size_t i = 0; i < max_iter; i++)
            table[i] = (uint32_t)std::uniform_int_distribution<size_t>(0, n * (i + 1) / max_iter + 1)(gen);
          const Expected e = restated(n, seed, target, max_iter, table);
          cases++;
          exits += e.iterations < max_iter;
          kept += e.have_best;
          for (const auto& s : schedules) {
            FakeModel m{table};
            cb::RansacRun r;
            cb::RansacSampler sampler(n, seed);
            const int rc = cb::ransac_loop(sampler, target, max_iter, s[0], s[1], m, &r);
            const char* fmt = "n=%zu target=%zu max_iter=%zu seed=%u schedule=(%zu,%zu): %s";
#define SAME(cond, what) CHECK(cond, fmt, n, target, max_iter, seed, s[0], s[1], what)
            SAME(rc == 0, "return code");
            SAME(r.sample_size == e.sample_size, "sample size clamp");
            SAME(r.target == e.target, "target clamp");
            SAME(r.iterations == e.iterations, "iterations");
            SAME(r.have_best == e.have_best, "have_best");
            SAME(r.best_count == e.best_count, "best count");
            SAME(!e.have_best || r.best_iteration == e.best_iteration, "best iteration");
            SAME(e.have_best ? m.kept == e.best_iteration : m.kept == SIZE_MAX, "kept hypothesis");
            SAME(m.samples.size() >= e.samples.size() &&
                     std::equal(e.samples.begin(), e.samples.end(), m.samples.begin()),
                 "sample sequence");
            // batch sizes: first, doubled up to max, the last cut at max_iter; none after the early exit
            size_t want = s[0], done = 0;
            bool ok = true;
            for (size_t nb : m.batches) {
              ok = ok && nb == std::min(want, max_iter - done);
              done += nb;
              want = std::min(2 * want, s[1]);
            }
            if (m.batches.empty())
              ok = ok && e.iterations == 0;
            else
              ok = ok && done >= e.iterations && done - m.batches.back() < e.iterations;
            SAME(ok, "batch schedule");
#undef SAME
          }
        }
  }
  // an error code from a hook ends the loop and is returned
  {
    const std::vector<uint32_t> table(100, 0u);
    FakeModel m{table, 1};
    cb::RansacRun r;
    cb::RansacSampler sampler(50, 3u);
    const int rc = cb::ransac_loop(sampler, 50, 100, 8, 8, m, &r);
    CHECK(rc == 7 && m.batches.size() == 2 && r.iterations == 8, "hook error: rc=%d batches=%zu iterations=%zu", rc,
          m.batches.size(), r.iterations);
  }
  std::printf("%zu cases (%zu early exits, %zu with a kept hypothesis) x %zu schedules\n", cases, exits, kept,
              sizeof(schedules) / sizeof(schedules[0]));
  if (failures) {
    std::printf("%d failures\n", failures);
    return 1;
  }
  std::printf("all ransac-loop checks passed\n");
  return 0;
}
