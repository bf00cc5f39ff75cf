// An a_star.cpp / dijkstra.cpp-style C++11 program on top of crb/reference_api.hpp: the demo's map built the way
// main() :247-286 builds it, then a_star_planning and dijkstra_star_planning under the reference's names, once per
// query and once batched.  Built with -Wall -Werror by tests/test_grid.py.
//   argv[1]: out.bin: for each planner the single-query demo path (length, then rx..., ry...), then for the batched
//            call over the queries (10, 10) -> (50, 50), (5, 55) -> (55, 5), (30, 30) -> (30, 30) each path the same way
#include <cstdio>
#include <vector>

#include "crb/reference_api.hpp"

using namespace std;
using namespace cpprobotics;

static void put(vector<float>& out, const vector<vector<float>>& p) {
  out.push_back((float)p[0].size());
  out.insert(out.end(), p[0].begin(), p[0].end());
  out.insert(out.end(), p[1].begin(), p[1].end());
}

int main(int argc, char** argv) {
  if (argc != 2) return 2;
  float sx = 10.0;
  float sy = 10.0;
  float gx = 50.0;
  float gy = 50.0;
  float grid_size = 1.0;
  float robot_size = 1.0;
  vector<float> ox;
  vector<float> oy;
  for (float i = 0; i < 60; i++) { ox.push_back(i); oy.push_back(60.0); }
  for (float i = 0; i < 60; i++) { ox.push_back(60.0); oy.push_back(i); }
  for (float i = 0; i < 61; i++) { ox.push_back(i); oy.push_back(60.0); }
  for (float i = 0; i < 61; i++) { ox.push_back(0.0); oy.push_back(i); }
  for (float i = 0; i < 40; i++) { ox.push_back(20.0); oy.push_back(i); }
  for (float i = 0; i < 40; i++) { ox.push_back(40.0); oy.push_back(60.0 - i); }

  a_star_planning(sx, sy, gx, gy, ox, oy, grid_size, robot_size);  // as the reference calls it: result ignored
  vector<float> out;
  put(out, a_star_planning(sx, sy, gx, gy, ox, oy, grid_size, robot_size));
  put(out, dijkstra_star_planning(sx, sy, gx, gy, ox, oy, grid_size, robot_size));
  vector<float> bsx = {10.0f, 5.0f, 30.0f}, bsy = {10.0f, 55.0f, 30.0f};
  vector<float> bgx = {50.0f, 55.0f, 30.0f}, bgy = {50.0f, 5.0f, 30.0f};
  for (int algo = 0; algo < 2; ++algo) {
    vector<vector<vector<float>>> ps = algo == 0 ? a_star_planning(bsx, bsy, bgx, bgy, ox, oy, grid_size, robot_size)
                                                 : dijkstra_star_planning(bsx, bsy, bgx, bgy, ox, oy, grid_size,
                                                                          robot_size);
    for (size_t i = 0; i < ps.size(); ++i) put(out, ps[i]);
  }
  FILE* o = std::fopen(argv[1], "wb");
  if (!o) return 2;
  std::fwrite(out.data(), sizeof(float), out.size(), o);
  std::fclose(o);
  return 0;
}
