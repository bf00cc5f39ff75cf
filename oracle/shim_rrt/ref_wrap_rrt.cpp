// oracle/shim_rrt/ref_wrap_rrt.cpp — C entry point around the reference's own include/rrt.h, #included from where it
// lies (nothing of it is copied into this repository).  A subclass of RRT seeds goal_gen in its constructor and exposes
// node_list after planning(); std::cout (the "find path" line) is silenced.
#include <cstdint>
#include <iostream>
#include <map>
#include <random>
#include <sstream>
#include <vector>

#include "rrt.h"

namespace {
struct SeededRRT : cpprobotics::RRT {
  SeededRRT(cpprobotics::Node* s, cpprobotics::Node* g, std::vector<std::vector<float> > ob, std::vector<float> area,
            float expand_dis, int goal_sample_rate, uint32_t seed)
      : cpprobotics::RRT(s, g, ob, area, expand_dis, 1.0f, goal_sample_rate, 500) {
    goal_gen.seed(seed);
  }
  const std::vector<cpprobotics::Node*>& nodes() const { return node_list; }
  // generator outputs consumed since seeding (at most cap)
  long long draws(uint32_t seed, long long cap) const {
    std::mt19937 m(seed);
    long long d = 0;
    while (!(m == goal_gen) && d < cap) {
      m();
      ++d;
    }
    return d;
  }
};
}  // namespace

extern "C" {
// RRT::planning for one query with goal_gen.seed(seed).  ob [n_ob][3] rows (x, y, r).  Returns the number of nodes in
// node_list, with node k at tree [2k], tree [2k + 1] and its parent's index (-1 for the start) at parent [k] for
// k < cap; the returned path's points (end ... start) at path [2j], path [2j + 1] for j < cap + 1 and their number in
// *path_len; the generator outputs consumed in *draws.  Returns -1, with nothing written, when the planner accepts
// more than cap nodes (it is only called for queries the checker finds reach the goal, so this bounds a checker bug).
int ref_rrt_run(float sx, float sy, float gx, float gy, int n_ob, const float* ob, float rand_min, float rand_max,
                float expand_dis, int goal_sample_rate, uint32_t seed, int cap, float* tree, int* parent, float* path,
                int* path_len, long long* draws) {
  std::vector<std::vector<float> > obs;
  for (int j = 0; j < n_ob; ++j) obs.push_back({ob[3 * j], ob[3 * j + 1], ob[3 * j + 2]});
  SeededRRT r(new cpprobotics::Node(sx, sy), new cpprobotics::Node(gx, gy), obs, {rand_min, rand_max}, expand_dis,
              goal_sample_rate, seed);
  std::streambuf* old = std::cout.rdbuf();
  std::ostringstream sink;
  std::cout.rdbuf(sink.rdbuf());
  cv::line_count() = 0;
  cv::line_limit() = 2L * cap + 2;  // one line per accepted node, then one per path segment
  std::vector<cpprobotics::Node*> p;
  bool ok = true;
  try {
    p = r.planning();
  } catch (const cv::LineLimit&) {
    ok = false;
  }
  std::cout.rdbuf(old);
  const std::vector<cpprobotics::Node*>& nl = r.nodes();
  if (!ok || (int)nl.size() > cap) return -1;
  std::map<const cpprobotics::Node*, int> index;
  for (size_t k = 0; k < nl.size(); ++k) index[nl[k]] = (int)k;
  for (size_t k = 0; k < nl.size(); ++k) {
    tree[2 * k] = nl[k]->x;
    tree[2 * k + 1] = nl[k]->y;
    parent[k] = nl[k]->parent ? index.at(nl[k]->parent) : -1;
  }
  for (size_t j = 0; j < p.size(); ++j) {
    path[2 * j] = p[j]->x;
    path[2 * j + 1] = p[j]->y;
  }
  *path_len = (int)p.size();
  *draws = r.draws(seed, 100000000LL);
  return (int)nl.size();
}
}
