// An rrt.cpp-style C++11 program on top of crb/reference_api.hpp: the demo's obstacles, start and goal built the way
// main() (src/rrt.cpp:17-38) builds them, then RRT::planning under the reference's names, seeded, once per query and
// once batched.  Built with -Wall -Werror by tests/test_rrt.py.
//   argv[1]: out.bin: for the single-query demo with goal_gen.seed(7) the path (length, then x, y of each point), then
//            for the batched call with seeds 1, 2, 3 and starts (0, 0), (12, 2), (6, 9) each path the same way
#include <cstdio>
#include <vector>

#include "crb/reference_api.hpp"

using namespace std;
using namespace cpprobotics;

static void put(vector<float>& out, const vector<Node*>& p) {
  out.push_back((float)p.size());
  for (size_t k = 0; k < p.size(); ++k) {
    if (k > 0 && k + 1 < p.size() && p[k]->parent != p[k + 1]) out.push_back(-1.0f);  // a broken parent chain
    out.push_back(p[k]->x);
    out.push_back(p[k]->y);
  }
}

int main(int argc, char** argv) {
  if (argc != 2) return 2;
  std::vector<vector<float> > obstacle_list{{5, 5, 1}, {3, 6, 2}, {3, 8, 2}, {3, 10, 2}, {7, 5, 2}, {9, 5, 2}};
  Node* start = new Node(0.0, 0.0);
  Node* goal = new Node(6.0, 9.0);
  std::vector<float> rand_area{-2, 15};
  RRT rrt(start, goal, obstacle_list, rand_area, 0.5);
  rrt.planning();  // seeded from std::random_device, as the reference is: result unused
  rrt.seed(7);
  vector<float> out;
  put(out, rrt.planning());
  vector<Node*> starts = {new Node(0, 0), new Node(12, 2), new Node(6, 9)};
  vector<Node*> goals = {new Node(6, 9), new Node(6, 9), new Node(6, 9)};
  vector<vector<Node*> > ps = rrt.planning(starts, goals, {1u, 2u, 3u});
  for (size_t i = 0; i < ps.size(); ++i) put(out, ps[i]);
  FILE* o = std::fopen(argv[1], "wb");
  if (!o) return 2;
  std::fwrite(out.data(), sizeof(float), out.size(), o);
  std::fclose(o);
  return 0;
}
