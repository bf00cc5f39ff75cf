// A state_lattice_planner-style C++11 program on top of crb/reference_api.hpp: the reference's Table, StateList,
// samplers, search_nearest_one_from_lookuptable and generate_path, used the way src/state_lattice_planner.cpp:157-231
// uses them.  Built with -Wall -Werror by tests/test_slp.py.
//   argv[1]: a lookup table as rows of 6 floats (binary, the rows already parsed); argv[2]: out.bin
//   out.bin: for each of the three demo scenarios the number of trajectories, then per trajectory its length and its
//            points (x, y, yaw); then the search result (distance, steering[0..2]) of the first uniform state
#include <cmath>
#include <cstdio>
#include <vector>

#include "crb/reference_api.hpp"

using namespace cpprobotics;

static void put(std::vector<float>& out, const std::vector<Traj>& ts) {
  out.push_back((float)ts.size());
  for (const Traj& t : ts) {
    out.push_back((float)t.size());
    for (const TrajState& s : t) {
      out.push_back(s.x);
      out.push_back(s.y);
      out.push_back(s.yaw);
    }
  }
}

std::vector<Traj> uniform_terminal_state_sample_test(Table csv_file) {
  float k0 = 0.0;
  int nxy = 5;
  int nh = 3;
  int d = 20;
  float a_min = -45.0 / 180 * M_PI;
  float a_max = +45.0 / 180 * M_PI;
  float p_min = -45.0 / 180 * M_PI;
  float p_max = +45.0 / 180 * M_PI;
  StateList states = calc_uniform_polar_states(nxy, nh, d, a_min, a_max, p_min, p_max);
  return generate_path(states, csv_file, k0);
}

std::vector<Traj> biased_terminal_state_sample_test(Table csv_file) {
  float k0 = 0.0;
  int nxy = 30;
  int nh = 2;
  int d = 20;
  float a_min = -45.0 / 180 * M_PI;
  float a_max = +45.0 / 180 * M_PI;
  float p_min = -20.0 / 180 * M_PI;
  float p_max = +20.0 / 180 * M_PI;
  int ns = 100;
  float goal_angle = 0.0;
  StateList states = calc_biased_polar_states(goal_angle, ns, nxy, nh, d, a_min, a_max, p_min, p_max);
  return generate_path(states, csv_file, k0);
}

std::vector<Traj> lane_state_sample_test(Table csv_file) {
  float k0 = 0.0;
  float l_center = 10.0;
  float l_heading = 90.0 / 180.0 * M_PI;
  float l_width = 3.0;
  float v_width = 1.0;
  int d = 10;
  int nxy = 5;
  StateList states = calc_lane_states(l_center, l_heading, l_width, v_width, d, nxy);
  return generate_path(states, csv_file, k0);
}

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 2;
  Table lookup_table;
  float row[6];
  while (std::fread(row, sizeof(float), 6, in) == 6) lookup_table.push_back(std::vector<float>(row, row + 6));
  std::fclose(in);
  std::vector<float> out;
  put(out, uniform_terminal_state_sample_test(lookup_table));
  put(out, biased_terminal_state_sample_test(lookup_table));
  put(out, lane_state_sample_test(lookup_table));
  StateList first = calc_uniform_polar_states(5, 3, 20, -45.0 / 180 * M_PI, 45.0 / 180 * M_PI, -45.0 / 180 * M_PI,
                                              45.0 / 180 * M_PI);
  Parameter p = search_nearest_one_from_lookuptable(first[0], lookup_table);
  out.push_back(p.distance);
  for (int k = 0; k < 3; ++k) out.push_back(p.steering_sequence[k]);
  FILE* o = std::fopen(argv[2], "wb");
  if (!o) return 2;
  std::fwrite(out.data(), sizeof(float), out.size(), o);
  std::fclose(o);
  return 0;
}
