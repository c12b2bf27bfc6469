// The RandomSampleConsensusBase surface (model_estimation/ransac_base.hpp) of both RANSAC drop-ins,
// RigidTransformRANSACEstimator3f<> and PlaneRANSACEstimator3f<>: estimate() clamps the sample size (:67) and the
// target inlier count (:68) to the number of data points on the object, so the getters and
// targetInlierCountAchieved() report the clamped values afterwards; the result getters come in both forms.
// tests/test_cpp_shims.py builds and runs it. Exit code 0 = all checks passed.
#include <cstdio>
#include <cstring>
#include <vector>

#include <cilantro/model_estimation/ransac_hyperplane_estimator.hpp>
#include <cilantro/model_estimation/ransac_transform_estimator.hpp>

static int failures = 0;
#define CHECK(cond)                                           \
  do {                                                        \
    if (!(cond)) {                                            \
      std::printf("FAIL line %d: %s\n", __LINE__, #cond);     \
      failures++;                                             \
    }                                                         \
  } while (0)

// the surface both estimators share, on n points where the model of every sample explains all n
template <class Estimator>
static void check_clamps(Estimator& e, size_t n) {
  CHECK(e.getSampleSize() == 3);
  CHECK(e.getTargetInlierCount() == n / 2 + n % 2);
  CHECK(e.getMaxNumberOfIterations() == 100);
  CHECK(e.getReEstimationStep());
  e.setTargetInlierCount(n + 5).setMaxNumberOfIterations(4).setReEstimationStep(false).setRandomSeed(3);
  CHECK(e.getTargetInlierCount() == n + 5);
  e.estimate();
  CHECK(e.getSampleSize() == (n < 3 ? n : 3));
  CHECK(e.getTargetInlierCount() == n);
  CHECK(e.getNumberOfInliers() == n);
  CHECK(e.targetInlierCountAchieved());
  CHECK(e.getNumberOfPerformedIterations() == 1);
  e.estimate(0.5f, 2 * n + 1, 7);  // the three-argument form sets, then clamps again
  CHECK(e.getMaxInlierResidual() == 0.5f && e.getMaxNumberOfIterations() == 7 && e.getTargetInlierCount() == n);
  typename Estimator::Model m;
  typename Estimator::ResidualVector r;
  typename Estimator::IndexVector i;
  e.getEstimationResults(m, r, i);
  CHECK(std::memcmp(&m, &e.getModel(), sizeof(m)) == 0 && r == e.getModelResiduals() && i == e.getModelInliers());
  typename Estimator::Model m2;
  e.getModel(m2).getModelResiduals(r).getModelInliers(i);
  CHECK(std::memcmp(&m2, &e.getModel(), sizeof(m2)) == 0 && r.size() == n && i.size() == n);
}

int main() {
  for (size_t n : {2, 40}) {
    // rigid: dst = src on the moment curve (no three points collinear), so every sample's fit is the identity
    cilantro::VectorSet3f pts(3, n);
    for (size_t k = 0; k < n; k++) {
      const float t = (float)k / 40.f;
      pts.setCol(k, cilantro::Vector3f(t, t * t, t * t * t));
    }
    cilantro::RigidTransformRANSACEstimator3f<> rigid(pts, pts);
    CHECK(rigid.getMaxInlierResidual() == 0.01f);
    check_clamps(rigid, n);
    // plane: a parabola in z = 0 (no three points collinear)
    cilantro::VectorSet3f flat(3, n);
    for (size_t k = 0; k < n; k++) {
      const float t = (float)k / 40.f;
      flat.setCol(k, cilantro::Vector3f(t, t * t, 0.f));
    }
    cilantro::PlaneRANSACEstimator3f<> plane(flat);
    CHECK(plane.getMaxInlierResidual() == 0.1f);
    check_clamps(plane, n);
  }
  if (failures) return 1;
  std::printf("all RANSAC clamp checks passed\n");
  return 0;
}
