// A dynamic_window_approach.cpp-style program on include/crb/reference_api.hpp: its own Config class and the
// reference's type aliases, dwa_control() and motion() called with the reference's signatures.
// Usage: dwa_ref_api in.bin out.bin
//   in:  float32 m, n_ob, then m robots of (x[5], u[2], goal[2]), then n_ob rows (ox, oy)
//   out: float32 per robot: u[2], n_pts, the returned trajectory (n_pts x 5), motion(x, u, config.dt)[5]
#include <array>
#include <cstdio>
#include <vector>

#include "crb/reference_api.hpp"

#define PI 3.141592653

using Traj = std::vector<std::array<float, 5>>;
using Obstacle = std::vector<std::array<float, 2>>;
using State = std::array<float, 5>;
using Point = std::array<float, 2>;
using Control = std::array<float, 2>;

class Config {
 public:
  float max_speed = 1.0;
  float min_speed = -0.5;
  float max_yawrate = 40.0 * PI / 180.0;
  float max_accel = 0.2;
  float robot_radius = 1.0;
  float max_dyawrate = 40.0 * PI / 180.0;
  float v_reso = 0.01;
  float yawrate_reso = 0.1 * PI / 180.0;
  float dt = 0.1;
  float predict_time = 3.0;
  float to_goal_cost_gain = 1.0;
  float speed_cost_gain = 1.0;
};

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 2;
  std::vector<float> buf;
  float v;
  while (std::fread(&v, sizeof(float), 1, in) == 1) buf.push_back(v);
  std::fclose(in);
  const int m = (int)buf[0], n_ob = (int)buf[1];
  const float* r = buf.data() + 2;
  Obstacle ob;
  for (int k = 0; k < n_ob; ++k) ob.push_back(Point{{r[9 * m + 2 * k], r[9 * m + 2 * k + 1]}});
  Config config;
  std::vector<float> out;
  try {
    for (int i = 0; i < m; ++i, r += 9) {
      State x = {{r[0], r[1], r[2], r[3], r[4]}};
      Control u = {{r[5], r[6]}};
      Point goal = {{r[7], r[8]}};
      Traj traj = dwa_control(x, u, config, goal, ob);
      State next = motion(x, u, config.dt);
      out.push_back(u[0]);
      out.push_back(u[1]);
      out.push_back((float)traj.size());
      for (size_t k = 0; k < traj.size(); ++k)
        for (int j = 0; j < 5; ++j) out.push_back(traj[k][j]);
      for (int j = 0; j < 5; ++j) out.push_back(next[j]);
    }
  } catch (const std::exception& e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 3;
  }
  FILE* o = std::fopen(argv[2], "wb");
  if (!o) return 2;
  std::fwrite(out.data(), sizeof(float), out.size(), o);
  std::fclose(o);
  return 0;
}
