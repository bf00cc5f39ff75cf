// An a_star.cpp / dijkstra.cpp-style C++11 program on top of crb/reference_api.hpp that plans every query on its own
// map: the demo's walls at robot radius 1 and 0.5, and a walled 20 m square at grid_size 0.5, through the overloads of
// a_star_planning and dijkstra_star_planning that take one obstacle list, grid size and robot size per query.  Built
// with -Wall -Werror by tests/test_grid_many_maps.py.
//   argv[1]: out.bin: for A*, then Dijkstra, each query's path (length, then rx..., ry...)
#include <cstdio>
#include <vector>

#include "crb/reference_api.hpp"

using namespace std;
using namespace cpprobotics;

int main(int argc, char** argv) {
  if (argc != 2) return 2;
  vector<float> ox;
  vector<float> oy;
  for (float i = 0; i < 60; i++) { ox.push_back(i); oy.push_back(60.0); }
  for (float i = 0; i < 60; i++) { ox.push_back(60.0); oy.push_back(i); }
  for (float i = 0; i < 61; i++) { ox.push_back(i); oy.push_back(60.0); }
  for (float i = 0; i < 61; i++) { ox.push_back(0.0); oy.push_back(i); }
  for (float i = 0; i < 40; i++) { ox.push_back(20.0); oy.push_back(i); }
  for (float i = 0; i < 40; i++) { ox.push_back(40.0); oy.push_back(60.0 - i); }
  vector<float> qx;
  vector<float> qy;
  for (float i = 0; i <= 20; i += 0.5f) {
    qx.push_back(i); qy.push_back(0.0f);
    qx.push_back(i); qy.push_back(20.0f);
    qx.push_back(0.0f); qy.push_back(i);
    qx.push_back(20.0f); qy.push_back(i);
  }
  vector<float> sx = {10.0f, 5.0f, 1.0f}, sy = {10.0f, 55.0f, 1.0f};
  vector<float> gx = {50.0f, 55.0f, 8.0f}, gy = {50.0f, 5.0f, 18.5f};
  vector<vector<float>> ox_ = {ox, ox, qx}, oy_ = {oy, oy, qy};
  vector<float> reso = {1.0f, 1.0f, 0.5f}, rr = {1.0f, 0.5f, 0.5f};
  vector<float> out;
  for (int algo = 0; algo < 2; ++algo) {
    vector<vector<vector<float>>> ps = algo == 0 ? a_star_planning(sx, sy, gx, gy, ox_, oy_, reso, rr)
                                                 : dijkstra_star_planning(sx, sy, gx, gy, ox_, oy_, reso, rr);
    for (size_t i = 0; i < ps.size(); ++i) {
      out.push_back((float)ps[i][0].size());
      out.insert(out.end(), ps[i][0].begin(), ps[i][0].end());
      out.insert(out.end(), ps[i][1].begin(), ps[i][1].end());
    }
  }
  FILE* o = std::fopen(argv[1], "wb");
  if (!o) return 2;
  std::fwrite(out.data(), sizeof(float), out.size(), o);
  std::fclose(o);
  return 0;
}
