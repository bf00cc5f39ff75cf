// A fleet of EKF localisers written against include/crb/reference_api.hpp: six robots in two sensor classes (a precise
// GPS with a well-known drive train, and a coarse GPS with a slipping one) run the demo's tick of
// src/extended_kalman_filter.cpp:171-183 for 50 steps, each with its own Q and R, through the fleet overload of
// ekf_estimation.  The program prints each robot's Q and R, its initial estimate, every tick's z and ud, and its
// final xEst and PEst as hex floats, and a checksum, so that a checker can recompute the run.
#include <cmath>
#include <cstdio>
#include <random>
#include <vector>

#include "crb/reference_api.hpp"

static void put(const char* name, const float* v, size_t n) {
  std::printf("%s", name);
  for (size_t i = 0; i < n; ++i) std::printf(" %a", (double)v[i]);
  std::printf("\n");
}

int main() {
  const int nr = 6, steps = 50;
  const float DT = 0.1f, PI = 3.141592653f;
  std::vector<crb::Vector4f> xEst(nr), xTrue(nr);
  std::vector<crb::Matrix4f> PEst(nr, crb::Matrix4f::Identity()), Q(nr, crb::Matrix4f::Identity());
  std::vector<crb::Matrix2f> R(nr, crb::Matrix2f::Identity());
  std::vector<crb::Vector2f> u(nr), ud(nr), z(nr);
  std::vector<float> gps(nr), slip(nr);
  for (int r = 0; r < nr; ++r) {
    const bool precise = r % 2 == 0;
    gps[r] = precise ? 0.2f : 1.0f;          // observation noise (the demo's Rsim)
    slip[r] = precise ? 0.3f : 1.0f;         // control noise (the demo's Qsim)
    Q[r](0, 0) = precise ? 0.05f * 0.05f : 0.2f * 0.2f;
    Q[r](1, 1) = Q[r](0, 0);
    Q[r](2, 2) = (1.0f / 180 * PI) * (1.0f / 180 * PI) * (precise ? 1.0f : 4.0f);
    Q[r](3, 3) = precise ? 0.05f * 0.05f : 0.2f * 0.2f;
    R[r](0, 0) = gps[r] * gps[r];
    R[r](1, 1) = gps[r] * gps[r];
    for (int k = 0; k < 4; ++k) xEst[r](k) = xTrue[r](k) = 0.0f;
    xTrue[r](0) = xEst[r](0) = 2.0f * (float)r;
    u[r](0) = 1.0f + 0.1f * (float)r;
    u[r](1) = 0.1f - 0.04f * (float)r;
  }
  std::printf("nr %d steps %d\n", nr, steps);
  for (int r = 0; r < nr; ++r) {
    put("Q", Q[r].data(), 16);
    put("R", R[r].data(), 4);
    put("x0", xEst[r].data(), 4);
    put("P0", PEst[r].data(), 16);
  }
  std::mt19937 gen(42);
  std::normal_distribution<> gaussian_d{0, 1};
  for (int t = 0; t < steps; ++t) {
    for (int r = 0; r < nr; ++r) {
      ud[r](0) = u[r](0) + (float)gaussian_d(gen) * slip[r];
      ud[r](1) = u[r](1) + (float)gaussian_d(gen) * slip[r] * (30.0f / 180 * PI);
      // the true pose follows the commanded input (motion_model :22-36 with v = u(0))
      const float yaw = xTrue[r](2);
      xTrue[r](0) += DT * std::cos(yaw) * u[r](0);
      xTrue[r](1) += DT * std::sin(yaw) * u[r](0);
      xTrue[r](2) += DT * u[r](1);
      z[r](0) = xTrue[r](0) + (float)gaussian_d(gen) * gps[r];
      z[r](1) = xTrue[r](1) + (float)gaussian_d(gen) * gps[r];
      put("z", z[r].data(), 2);
      put("ud", ud[r].data(), 2);
    }
    ekf_estimation(xEst, PEst, z, ud, Q, R);
  }
  double checksum = 0.0;
  for (int r = 0; r < nr; ++r) {
    put("xEst", xEst[r].data(), 4);
    put("PEst", PEst[r].data(), 16);
    for (int k = 0; k < 4; ++k) checksum += xEst[r](k);
  }
  std::printf("checksum %.9e\n", checksum);
  return 0;
}
