// oracle/shim/ref_wrap_slp.cpp — C entry points around the reference's own src/state_lattice_planner.cpp.  The file
// is #included from where it lies (REF_SRC, set by oracle/Makefile) with main() renamed; nothing of it is copied into
// this repository.  <limits> comes first: the file and the headers it includes use std::numeric_limits and rely on
// real OpenCV's headers to include it.
#include <limits>

#define main crb_reference_main
#include REF_SRC
#undef main

namespace {
// a StateList as rows (x, y, yaw); the list's full size is returned, at most cap rows are copied
int put_states(const StateList& s, float* out, int cap) {
  for (size_t k = 0; k < s.size() && (int)k < cap; ++k) {
    out[3 * k] = s[k].x;
    out[3 * k + 1] = s[k].y;
    out[3 * k + 2] = s[k].yaw;
  }
  return (int)s.size();
}
Table table_of(const float* t, int rows) {
  Table tb;
  for (int r = 0; r < rows; ++r) tb.push_back(std::vector<float>(t + 6 * r, t + 6 * r + 6));
  return tb;
}
// trajectories as rows of (x, y, yaw), max_pts per trajectory (NaN beyond its end is the caller's), and lengths
void put_trajs(const std::vector<Traj>& ts, float* traj, int max_pts, int* len) {
  for (size_t i = 0; i < ts.size(); ++i) {
    len[i] = (int)ts[i].size();
    for (size_t k = 0; k < ts[i].size() && (int)k < max_pts; ++k) {
      traj[3 * (i * max_pts + k)] = ts[i][k].x;
      traj[3 * (i * max_pts + k) + 1] = ts[i][k].y;
      traj[3 * (i * max_pts + k) + 2] = ts[i][k].yaw;
    }
  }
}
}  // namespace

extern "C" {
int ref_slp_uniform(int nxy, int nh, int d, float a_min, float a_max, float p_min, float p_max, float* out, int cap) {
  return put_states(calc_uniform_polar_states(nxy, nh, d, a_min, a_max, p_min, p_max), out, cap);
}
int ref_slp_biased(float goal_angle, int ns, int nxy, int nh, int d, float a_min, float a_max, float p_min,
                   float p_max, float* out, int cap) {
  return put_states(calc_biased_polar_states(goal_angle, ns, nxy, nh, d, a_min, a_max, p_min, p_max), out, cap);
}
int ref_slp_lane(float l_center, float l_heading, float l_width, float v_width, float d, int nxy, float* out,
                 int cap) {
  return put_states(calc_lane_states(l_center, l_heading, l_width, v_width, d, nxy), out, cap);
}
// search_nearest_one_from_lookuptable for n targets (rows of x, y, yaw); param rows (distance, steering[0..2])
void ref_slp_search(int n, const float* target, const float* table, int rows, float* param) {
  const Table tb = table_of(table, rows);
  for (int i = 0; i < n; ++i) {
    Parameter p = search_nearest_one_from_lookuptable(TrajState(target[3 * i], target[3 * i + 1], target[3 * i + 2]),
                                                      tb);
    param[4 * i] = p.distance;
    for (int k = 0; k < 3; ++k) param[4 * i + 1 + k] = p.steering_sequence[k];
  }
}
// generate_path(states, table, k0) for n states
void ref_slp_generate_path(int n, const float* states, const float* table, int rows, float k0, float* traj,
                           int max_pts, int* len) {
  StateList s;
  for (int i = 0; i < n; ++i) s.push_back(TrajState(states[3 * i], states[3 * i + 1], states[3 * i + 2]));
  put_trajs(generate_path(s, table_of(table, rows), k0), traj, max_pts, len);
}
// the demo's three scenarios (:157-210) on a table: which = 0 uniform, 1 biased, 2 lane; returns the number of
// trajectories (at most cap are copied)
int ref_slp_demo(int which, const float* table, int rows, float* traj, int max_pts, int* len, int cap) {
  const Table tb = table_of(table, rows);
  std::vector<Traj> ts = which == 0 ? uniform_terminal_state_sample_test(tb)
                         : which == 1 ? biased_terminal_state_sample_test(tb)
                                      : lane_state_sample_test(tb);
  const int n = (int)ts.size();
  if ((int)ts.size() > cap) ts.resize((size_t)cap);
  put_trajs(ts, traj, max_pts, len);
  return n;
}
// main()'s reading of the table (:214-226): CSVIterator, the header row skipped, std::stod of 6 fields narrowed to
// float.  Returns the number of rows (at most cap copied), or -1 when a field does not parse (stod throws).
int ref_slp_read_csv(const char* path, float* out, int cap) {
  std::vector<std::vector<float>> lookup_table;
  std::ifstream file(path);
  CSVIterator loop(file);
  loop++;
  try {
    for (; loop != CSVIterator(); ++loop) {
      std::vector<float> temp;
      for (int i = 0; i < 6; i++) {
        temp.push_back(std::stod((*loop)[i]));
      }
      lookup_table.push_back(temp);
    }
  } catch (const std::exception&) {
    return -1;
  }
  for (size_t r = 0; r < lookup_table.size() && (int)r < cap; ++r)
    for (int c = 0; c < 6; ++c) out[6 * r + c] = lookup_table[r][c];
  return (int)lookup_table.size();
}
}
