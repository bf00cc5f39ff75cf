// oracle/shim_grid/ref_wrap_grid.cpp — C entry point around the reference's own src/a_star.cpp or src/dijkstra.cpp (one
// library each: both files define Node and calc_final_path).  The file is #included from where it lies (REF_SRC, set
// by oracle/grid.mk) with main() renamed; nothing of it is copied into this repository.  REF_PLAN names the planner
// (a_star_planning or dijkstra_star_planning).
//
// The planners return nothing; everything they compute is drawn with cv::rectangle, which oracle/shim_grid's OpenCV
// stand-in hands to a recorder.  ref_grid_run records every call as (x1, y1, x2, y2, b, g, r, thickness): the start (blue) and goal (red)
// markers, the obstacle map (black, filled, box-relative cells), the expansion trace (green, outlined, absolute cells,
// in order) and calc_final_path's path (blue, filled, absolute cells, goal first).
#include <vector>

#define main crb_reference_main
#include REF_SRC
#undef main

namespace {
std::vector<int>* g_rec = nullptr;
void record(int x1, int y1, int x2, int y2, const cv::Scalar& c, int thickness) {
  const int v[8] = {x1, y1, x2, y2, (int)c.v[0], (int)c.v[1], (int)c.v[2], thickness};
  g_rec->insert(g_rec->end(), v, v + 8);
}
}  // namespace

extern "C" {
// runs the planner on (sx, sy, gx, gy, ox, oy, reso, rr); returns the number of calls (at most cap are copied into
// out [8 * cap]).  Only for inputs where the reference is defined: the caller checks that first.
int ref_grid_run(float sx, float sy, float gx, float gy, int n_obs, const float* ox, const float* oy, float reso,
                 float rr, int* out, int cap) {
  std::vector<int> rec;
  g_rec = &rec;
  cv::rectangle_recorder() = record;
  REF_PLAN(sx, sy, gx, gy, std::vector<float>(ox, ox + n_obs), std::vector<float>(oy, oy + n_obs), reso, rr);
  cv::rectangle_recorder() = nullptr;
  g_rec = nullptr;
  const int n = (int)(rec.size() / 8);
  for (int i = 0; i < 8 * n && i < 8 * cap; ++i) out[i] = rec[i];
  return n;
}
}
