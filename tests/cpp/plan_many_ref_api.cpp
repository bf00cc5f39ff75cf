// A fleet that plans among its own obstacles, written against include/crb/reference_api.hpp: dwa_control over a vector
// of robots with one obstacle list per robot, and RRT::planning with one obstacle list per query, each in one launch.
// Built with -Wall -Werror by tests/test_plan_many_obstacles.py.
// Usage: plan_many_ref_api in.bin out.bin
//   in:  float32 m, then m robots of (x[5], u[2], goal[2], k, k rows (ox, oy)); then q, then q queries of (sx, sy, gx,
//        gy, seed (uint32 bits), k, k rows (x, y, r)).  DWA runs with dynamic_window_approach.cpp's Config, RRT with
//        the demo's rand_area {-2, 15} and expand_dis 0.5.
//   out: float32 per robot: u[2], n_pts, the returned trajectory (n_pts x 5); per query: the path's length, then the
//        x, y of each point
#include <array>
#include <cstdio>
#include <cstring>
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

using namespace cpprobotics;

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
  std::vector<std::vector<std::array<float, 2>>> ob(m);
  for (int i = 0; i < m; ++i) {
    for (int f = 0; f < 5; ++f) x[i][f] = *r++;
    for (int f = 0; f < 2; ++f) u[i][f] = *r++;
    for (int f = 0; f < 2; ++f) goal[i][f] = *r++;
    const int k = (int)*r++;
    for (int j = 0; j < k; ++j, r += 2) ob[i].push_back(std::array<float, 2>{{r[0], r[1]}});
  }
  const int q = (int)*r++;
  std::vector<Node*> starts, ends;
  std::vector<uint32_t> seeds(q);
  std::vector<std::vector<std::vector<float> > > ob_lists(q);
  for (int i = 0; i < q; ++i) {
    starts.push_back(new Node(r[0], r[1]));
    ends.push_back(new Node(r[2], r[3]));
    std::memcpy(&seeds[i], &r[4], 4);
    const int k = (int)r[5];
    r += 6;
    for (int j = 0; j < k; ++j, r += 3) ob_lists[i].push_back(std::vector<float>{r[0], r[1], r[2]});
  }
  std::vector<float> out;
  try {
    std::vector<std::vector<std::array<float, 5>>> traj = dwa_control(x, u, Config(), goal, ob);
    for (int i = 0; i < m; ++i) {
      out.push_back(u[i][0]);
      out.push_back(u[i][1]);
      out.push_back((float)traj[i].size());
      for (size_t k = 0; k < traj[i].size(); ++k)
        for (int j = 0; j < 5; ++j) out.push_back(traj[i][k][j]);
    }
    std::vector<std::vector<float> > none;
    std::vector<float> rand_area{-2, 15};
    RRT rrt(new Node(0.0, 0.0), new Node(6.0, 9.0), none, rand_area, 0.5);
    std::vector<std::vector<Node*> > paths = rrt.planning(starts, ends, seeds, ob_lists);
    for (int i = 0; i < q; ++i) {
      out.push_back((float)paths[i].size());
      for (size_t k = 0; k < paths[i].size(); ++k) {
        out.push_back(paths[i][k]->x);
        out.push_back(paths[i][k]->y);
      }
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
