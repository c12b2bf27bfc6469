// Depth frames -> clouds -> registration, on the device: a synthetic room (a wall with relief, a floor and a box) is
// rendered from two camera poses with pointsToDepthImage, each 640 x 480 depth frame is converted back to points with
// organised normals (PointCloud3f's depth-image constructor), downsampled, given kNN normals and registered with
// SimpleCombinedMetricRigidICP3f. Prints the error of the recovered pose against the true one.
//
//   depth_image_cloud [cloud.ply]   (a PLY cloud, e.g. tests/golden/scan_excerpt.ply, replaces the synthetic room; it
//                                    is centred and placed 2.5 m in front of the first camera)
#include <cilantro/core/image_point_cloud_conversions.hpp>
#include <cilantro/registration/icp_common_instances.hpp>
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
    switch (i % 3) {
      case 0: {  // wall
        const float x = -2.f + 4.f * a, y = -1.5f + 3.f * b;
        p.setCol(i, {x, y, 4.f + 0.15f * std::sin(3.f * x) * std::cos(2.f * y)});
        break;
      }
      case 1:  // floor
        p.setCol(i, {-2.f + 4.f * a, 1.f, 1.5f + 2.5f * b});
        break;
      default: {  // three faces of a box
        const float u = -0.4f + 0.8f * a, v = -0.4f + 0.8f * b;
        const int face = (int)(i / 3) % 3;
        const cilantro::Vector3f q = face == 0 ? cilantro::Vector3f(u, v, -0.4f)
                                     : face == 1 ? cilantro::Vector3f(-0.4f, u, v)
                                                 : cilantro::Vector3f(u, -0.4f, v);
        p.setCol(i, {q[0] + 0.5f, q[1] + 0.4f, q[2] + 2.8f});
      }
    }
  }
  return p;
}

int main(int argc, char** argv) {
  const size_t w = 640, h = 480;
  const cilantro::b200::Intrinsics3f K(525.f, 525.f, 319.5f, 239.5f);
  cilantro::VectorSet3f scene;
  if (argc >= 2) {
    const cilantro::PointCloud3f ply(argv[1]);
    float c[3] = {0.f, 0.f, 0.f};
    for (size_t i = 0; i < ply.size(); i++)
      for (int r = 0; r < 3; r++) c[r] += ply.points(r, i) / (float)ply.size();
    scene.resize(3, ply.size());
    for (size_t i = 0; i < ply.size(); i++)
      scene.setCol(i, {ply.points(0, i) - c[0], ply.points(1, i) - c[1], ply.points(2, i) - c[2] + 2.5f});
  } else {
    scene = room(600000, 7);
  }
  // the second camera: 0.6 degrees about a tilted axis and a 2 cm shift
  cilantro::RigidTransform3f pose;
  const float ang = 0.0105f, ax[3] = {0.3f, 0.9f, 0.3f};
  const float nrm = std::sqrt(ax[0] * ax[0] + ax[1] * ax[1] + ax[2] * ax[2]);
  const float k[3] = {ax[0] / nrm, ax[1] / nrm, ax[2] / nrm}, s = std::sin(ang), c1 = 1.f - std::cos(ang);
  const float Kx[3][3] = {{0, -k[2], k[1]}, {k[2], 0, -k[0]}, {-k[1], k[0], 0}};
  for (int r = 0; r < 3; r++)
    for (int q = 0; q < 3; q++) {
      float kk = 0.f;
      for (int m = 0; m < 3; m++) kk += Kx[r][m] * Kx[m][q];
      pose.linear(r, q) = (r == q ? 1.f : 0.f) + s * Kx[r][q] + c1 * kk;
    }
  pose.translation(0) = 0.02f;
  pose.translation(1) = -0.01f;
  pose.translation(2) = 0.015f;

  const cilantro::DepthValueConverter<unsigned short, float> conv(1000.f);
  std::vector<unsigned short> depth_a(w * h), depth_b(w * h);
  cilantro::pointsToDepthImage(scene, K, conv, depth_a.data(), w, h);
  cilantro::pointsToDepthImage(scene, pose, K, conv, depth_b.data(), w, h);
  cilantro::PointCloud3f dst(depth_a.data(), conv, w, h, K, false, true);
  cilantro::PointCloud3f src(depth_b.data(), conv, w, h, K, false, true);
  std::printf("frames: %zu / %zu points with image normals\n", dst.size(), src.size());
  if (dst.isEmpty() || src.isEmpty()) return 1;

  dst.gridDownsample(0.02f);
  src.gridDownsample(0.02f);
  dst.estimateNormalsKNN(10);
  cilantro::SimpleCombinedMetricRigidICP3f icp(dst.points, dst.normals, src.points);
  icp.setMaxNumberOfOptimizationStepIterations(1).setPointToPointMetricWeight(0.1f).setPointToPlaneMetricWeight(1.0f);
  icp.correspondenceSearchEngine().setMaxDistance(0.1f * 0.1f);
  icp.setConvergenceTolerance(1e-6f).setMaxNumberOfIterations(50);
  const cilantro::RigidTransform3f T = icp.estimate().getTransform();
  std::printf("ICP: %zu / %zu points, %zu iterations\n", dst.size(), src.size(), icp.getNumberOfPerformedIterations());
  // src = pose^-1 applied to the scene of dst, so T should equal pose
  const cilantro::RigidTransform3f back = T * pose.inverse();
  float err = 0.f;
  for (int r = 0; r < 3; r++) {
    for (int q = 0; q < 3; q++) err += (back.linear(r, q) - (r == q)) * (back.linear(r, q) - (r == q));
    err += back.translation(r) * back.translation(r);
  }
  std::printf("Pose error |T * pose^-1 - I|_F: %.3e\n", std::sqrt(err));
  return (argc >= 2 || std::sqrt(err) < 1e-2f) ? 0 : 2;  // a scan excerpt may see too little to register
}
