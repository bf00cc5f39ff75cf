// A model_predictive_trajectory_generator-style C++11 program on top of crb/reference_api.hpp: the reference's
// State, TrajState, Parameter, MotionModel and TrajectoryOptimizer, used the way
// src/model_predictive_trajectory_generator.cpp:25-37 uses them.  Built with -Wall -Werror by tests/test_mptg.py.
//   in.bin : float m, then m records (state x y yaw v, target x y yaw, distance, steering[3])
//   out.bin: per record the optimised parameter [4], the trajectory length, its points [3 * len], then
//            generate_last_state of the optimised parameter [3]
#include <array>
#include <cstdio>
#include <vector>

#include "crb/reference_api.hpp"

#define L 1.0
#define DS 0.1

using namespace cpprobotics;

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 2;
  float mf = 0.0f;
  if (std::fread(&mf, sizeof(float), 1, in) != 1) return 2;
  const int m = (int)mf;
  std::vector<float> rec(11 * (size_t)m);
  if (std::fread(rec.data(), sizeof(float), rec.size(), in) != rec.size()) return 2;
  std::fclose(in);
  std::vector<float> out;
  for (int i = 0; i < m; ++i) {
    const float* r = &rec[11 * (size_t)i];
    State init_state(r[0], r[1], r[2], r[3]);
    TrajState target_(r[4], r[5], r[6]);
    MotionModel m_model(L, DS, init_state);
    Parameter p_(r[7], {{r[8], r[9], r[10]}});
    float cost_th_ = 0.1;
    std::vector<float> h_step_{0.2, 0.005, 0.005};
    int max_iter = 100;
    TrajectoryOptimizer traj_opti_obj(m_model, p_, target_);
    Traj traj = traj_opti_obj.optimizer_traj(max_iter, cost_th_, h_step_);
    const Parameter& p = traj_opti_obj.p;
    out.push_back(p.distance);
    for (int k = 0; k < 3; ++k) out.push_back(p.steering_sequence[k]);
    out.push_back((float)traj.size());
    for (const TrajState& s : traj) {
      out.push_back(s.x);
      out.push_back(s.y);
      out.push_back(s.yaw);
    }
    const TrajState last = m_model.generate_last_state(p);
    out.push_back(last.x);
    out.push_back(last.y);
    out.push_back(last.yaw);
  }
  FILE* o = std::fopen(argv[2], "wb");
  if (!o) return 2;
  std::fwrite(out.data(), sizeof(float), out.size(), o);
  std::fclose(o);
  return 0;
}
