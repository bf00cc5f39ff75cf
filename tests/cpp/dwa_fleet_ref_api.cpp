// A mixed fleet planned with the dynamic window approach, written against include/crb/reference_api.hpp: dwa_control
// over a vector of robots with a Config and an obstacle list per robot, then motion with each robot's config.dt, as
// src/dynamic_window_approach.cpp's main() does for one robot.  The same fleet is also planned with one Config
// (robot 0's) through the single-Config overload.  Built with -std=c++11 -Wall -Werror by tests/test_dwa_fleet.py.
// Usage: dwa_fleet_ref_api in.bin out.bin
//   in:  float32 m, then m robots of (x[5], u[2], goal[2], Config's twelve members in declaration order, k, k rows
//        (ox, oy))
//   out: float32 per robot: u[2], n_pts, the returned trajectory (n_pts x 5), the next state x[5]; then per robot the
//        u[2] of the single-Config call
#include <array>
#include <cstdio>
#include <vector>

#include "crb/reference_api.hpp"

#define PI 3.141592653

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
  const float* r = buf.data();
  const int m = (int)*r++;
  std::vector<std::array<float, 5>> x(m);
  std::vector<std::array<float, 2>> u(m), goal(m);
  std::vector<Config> config(m);
  std::vector<std::vector<std::array<float, 2>>> ob(m);
  for (int i = 0; i < m; ++i) {
    for (int f = 0; f < 5; ++f) x[i][f] = *r++;
    for (int f = 0; f < 2; ++f) u[i][f] = *r++;
    for (int f = 0; f < 2; ++f) goal[i][f] = *r++;
    Config& c = config[i];
    c.max_speed = *r++;
    c.min_speed = *r++;
    c.max_yawrate = *r++;
    c.max_accel = *r++;
    c.robot_radius = *r++;
    c.max_dyawrate = *r++;
    c.v_reso = *r++;
    c.yawrate_reso = *r++;
    c.dt = *r++;
    c.predict_time = *r++;
    c.to_goal_cost_gain = *r++;
    c.speed_cost_gain = *r++;
    const int k = (int)*r++;
    for (int j = 0; j < k; ++j, r += 2) ob[i].push_back(std::array<float, 2>{{r[0], r[1]}});
  }
  std::vector<float> out;
  try {
    std::vector<std::array<float, 2>> u_one = u;
    std::vector<std::vector<std::array<float, 5>>> traj = dwa_control(x, u, config, goal, ob);
    std::vector<float> dt(m);
    for (int i = 0; i < m; ++i) dt[i] = config[i].dt;
    const std::vector<std::array<float, 5>> next = motion(x, u, dt);
    for (int i = 0; i < m; ++i) {
      out.push_back(u[i][0]);
      out.push_back(u[i][1]);
      out.push_back((float)traj[i].size());
      for (size_t k = 0; k < traj[i].size(); ++k)
        for (int j = 0; j < 5; ++j) out.push_back(traj[i][k][j]);
      for (int f = 0; f < 5; ++f) out.push_back(next[i][f]);
    }
    dwa_control(x, u_one, config[0], goal, ob);
    for (int i = 0; i < m; ++i) {
      out.push_back(u_one[i][0]);
      out.push_back(u_one[i][1]);
    }
  } catch (const std::exception& e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 1;
  }
  FILE* o = std::fopen(argv[2], "wb");
  if (!o) return 2;
  std::fwrite(out.data(), sizeof(float), out.size(), o);
  std::fclose(o);
  return 0;
}
