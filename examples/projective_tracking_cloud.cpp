// Frame-to-model tracking with projective ICP, on the device: the localisation loop of the reference's fusion example
// without a viewer. A synthetic room (walls, floor and a box) is rendered along a camera trajectory with
// pointsToDepthImage, each 640 x 480 depth frame is converted back to points with organised normals, and every frame is
// tracked against the first frame's cloud with SimpleCombinedMetricRigidProjectiveICP3f and the fusion example's
// settings: the previous pose as the projection's extrinsics and the initial transform, max distance 0.1^2, 6
// iterations of one Gauss-Newton step, tolerance 5e-4. Prints the pose error of every frame.
#include <cilantro/core/image_point_cloud_conversions.hpp>
#include <cilantro/correspondence_search/correspondence_search_projective.hpp>
#include <cilantro/utilities/point_cloud.hpp>

#include <cmath>
#include <cstdio>
#include <random>
#include <vector>

static cilantro::VectorSet3f room(size_t n, unsigned seed) {
  std::mt19937 rng(seed);
  std::uniform_real_distribution<float> U(0.f, 1.f);
  cilantro::VectorSet3f p(3, n);
  for (size_t i = 0; i < n; i++) {
    const float a = U(rng), b = U(rng);
    switch (i % 5) {
      case 0:  // back wall
        p.setCol(i, {-2.f + 4.f * a, -1.5f + 3.f * b, 4.f});
        break;
      case 1:  // floor
        p.setCol(i, {-2.f + 4.f * a, 1.f, 0.5f + 3.5f * b});
        break;
      case 2:  // left wall
        p.setCol(i, {-2.f, -1.5f + 2.5f * a, 0.5f + 3.5f * b});
        break;
      case 3:  // right wall
        p.setCol(i, {2.f, -1.5f + 2.5f * a, 0.5f + 3.5f * b});
        break;
      default: {  // three faces of a box
        const float u = -0.4f + 0.8f * a, v = -0.4f + 0.8f * b;
        const int face = (int)(i / 5) % 3;
        const cilantro::Vector3f q = face == 0 ? cilantro::Vector3f(u, v, -0.4f)
                                     : face == 1 ? cilantro::Vector3f(-0.4f, u, v)
                                                 : cilantro::Vector3f(u, -0.4f, v);
        p.setCol(i, {q[0] + 0.5f, q[1] + 0.6f, q[2] + 2.8f});
      }
    }
  }
  return p;
}

// camera pose of frame k: a slow turn about a tilted axis and a drift
static cilantro::RigidTransform3f trajectory(int k) {
  cilantro::RigidTransform3f pose;
  const float ang = 0.004f * k, ax[3] = {0.2f, 0.95f, 0.25f};
  const float nrm = std::sqrt(ax[0] * ax[0] + ax[1] * ax[1] + ax[2] * ax[2]);
  const float u[3] = {ax[0] / nrm, ax[1] / nrm, ax[2] / nrm}, s = std::sin(ang), c1 = 1.f - std::cos(ang);
  const float Kx[3][3] = {{0, -u[2], u[1]}, {u[2], 0, -u[0]}, {-u[1], u[0], 0}};
  for (int r = 0; r < 3; r++)
    for (int q = 0; q < 3; q++) {
      float kk = 0.f;
      for (int m = 0; m < 3; m++) kk += Kx[r][m] * Kx[m][q];
      pose.linear(r, q) = (r == q ? 1.f : 0.f) + s * Kx[r][q] + c1 * kk;
    }
  pose.translation(0) = 0.01f * k;
  pose.translation(1) = -0.004f * k;
  pose.translation(2) = 0.015f * k;
  return pose;
}

int main() {
  const size_t w = 640, h = 480;
  const cilantro::b200::Intrinsics3f K(528.f, 528.f, 320.f, 240.f);
  const cilantro::VectorSet3f scene = room(1500000, 11);
  const cilantro::DepthValueConverter<unsigned short, float> conv(1000.f);
  std::vector<unsigned short> depth(w * h);

  // the model: the first frame's cloud with image normals (its camera is the world frame)
  cilantro::pointsToDepthImage(scene, trajectory(0), K, conv, depth.data(), w, h);
  const cilantro::PointCloud3f model(depth.data(), conv, w, h, K, false, true);
  std::printf("model: %zu points with image normals\n", model.size());
  if (model.isEmpty()) return 1;

  cilantro::RigidTransform3f cam_pose = trajectory(0);
  float worst = 0.f;
  const int frames = 10;
  for (int k = 1; k < frames; k++) {
    const cilantro::RigidTransform3f truth = trajectory(k);
    cilantro::pointsToDepthImage(scene, truth, K, conv, depth.data(), w, h);
    const cilantro::PointCloud3f frame(depth.data(), conv, w, h, K, false, true);

    cilantro::SimpleCombinedMetricRigidProjectiveICP3f icp(model.points, model.normals, frame.points, frame.normals);
    icp.correspondenceSearchEngine().setProjectionExtrinsicMatrix(cam_pose).setMaxDistance(0.1f * 0.1f)
        .setProjectionImageWidth(w).setProjectionImageHeight(h).setProjectionIntrinsicMatrix(K);
    icp.setInitialTransform(cam_pose).setConvergenceTolerance(5e-4f);
    icp.setMaxNumberOfIterations(6).setMaxNumberOfOptimizationStepIterations(1);
    cam_pose = icp.estimate().getTransform();

    const cilantro::RigidTransform3f back = cam_pose * truth.inverse();
    float err = 0.f;
    for (int r = 0; r < 3; r++) {
      for (int q = 0; q < 3; q++) err += (back.linear(r, q) - (r == q)) * (back.linear(r, q) - (r == q));
      err += back.translation(r) * back.translation(r);
    }
    err = std::sqrt(err);
    worst = std::fmax(worst, err);
    std::printf("frame %d: %zu points, %zu iterations, %zu correspondences, pose error |T * pose^-1 - I|_F = %.3e\n", k,
                frame.size(), icp.getNumberOfPerformedIterations(), icp.getCorrespondences().size(), err);
  }
  std::printf("worst pose error over %d frames: %.3e\n", frames - 1, worst);
  return worst < 1e-2f ? 0 : 2;
}
