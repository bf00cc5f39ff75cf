// A program shaped like closed_loop_prediction() of src/lqr_steer_control.cpp and src/lqr_speed_steer_control.cpp,
// written against include/crb/reference_api.hpp: the same calls with the reference's argument types, the loop kept by
// the caller with a tick cap (the reference's `while (T >= time_)` never advances time_).  The course is a quarter
// circle sampled every 0.1 m.  Prints each program's final state.
#include <cmath>
#include <cstdio>
#include <vector>

#include "crb/reference_api.hpp"

using namespace cpprobotics;

int main() {
  Vec_f cx, cy, cyaw, ck, sp;
  const float r = 10.0f, target_speed = 10.0f / 3.6f;
  for (float s = 0.0f; s < r * 1.5f; s += 0.1f) {
    cx.push_back(r * std::sin(s / r));
    cy.push_back(r - r * std::cos(s / r));
    cyaw.push_back(s / r);
    ck.push_back(1.0f / r);
    sp.push_back(target_speed);
  }
  sp.back() = 0.0f;
  const float goal_dis = 0.5f, stop_speed = 0.05f, KP = 1.0f;
  {
    State state(-0.0f, -0.0f, 0.0f, 0.0f);
    float e = 0, e_th = 0;
    int ind = 0;
    for (int tick = 0; tick < 600; ++tick) {
      float di = lqr_steer_control::lqr_steering_control(state, cx, cy, cyaw, ck, ind, e, e_th);
      float ai = KP * (sp[ind] - state.v);
      lqr_steer_control::update(state, ai, di);
      if (std::abs(state.v) <= stop_speed) ind += 1;
      float dx = state.x - cx.back();
      float dy = state.y - cy.back();
      if (std::sqrt(dx * dx + dy * dy) <= goal_dis) break;
    }
    std::printf("lqr_steer_control %.6f %.6f %.6f %.6f\n", state.x, state.y, state.yaw, state.v);
  }
  {
    State state(-0.0f, -0.0f, 0.0f, 0.0f);
    float e = 0, e_th = 0;
    for (int tick = 0; tick < 600; ++tick) {
      Vec_f control = lqr_speed_steer_control::lqr_steering_control(state, cx, cy, cyaw, ck, sp, e, e_th);
      lqr_speed_steer_control::update(state, control[0], control[1]);
      float dx = state.x - cx.back();
      float dy = state.y - cy.back();
      if (std::sqrt(dx * dx + dy * dy) <= goal_dis) break;
    }
    std::printf("lqr_speed_steer_control %.6f %.6f %.6f %.6f\n", state.x, state.y, state.yaw, state.v);
  }
  // a fleet in one call
  std::vector<State> fleet(8, State(0.0f, 0.5f, 0.1f, 1.0f));
  std::vector<int> ind(8, 0);
  Vec_f pe(8, 0.0f), pth_e(8, 0.0f);
  Vec_f delta = lqr_steer_control::lqr_steering_control(fleet, cx, cy, cyaw, ck, ind, pe, pth_e);
  lqr_steer_control::update(fleet, Vec_f(8, 0.5f), delta);
  std::printf("fleet %.6f\n", fleet[0].yaw);
  return 0;
}
