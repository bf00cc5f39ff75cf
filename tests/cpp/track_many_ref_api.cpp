// A fleet on many courses written against include/crb/reference_api.hpp: each vehicle follows its own quarter circle
// (radius 5 + i, sampled every 0.1 m) through the batched overloads that take one course per vehicle, with the loop
// kept by the caller.  Prints the first and last vehicle's final state for each program.
#include <cmath>
#include <cstdio>
#include <vector>

#include "crb/reference_api.hpp"

using namespace cpprobotics;

int main() {
  const int n = 6;
  std::vector<Vec_f> cx(n), cy(n), cyaw(n), ck(n), sp(n);
  for (int i = 0; i < n; ++i) {
    const float r = 5.0f + (float)i;
    for (float s = 0.0f; s < r * 1.5f; s += 0.1f) {
      cx[i].push_back(r * std::sin(s / r));
      cy[i].push_back(r - r * std::cos(s / r));
      cyaw[i].push_back(s / r);
      ck[i].push_back(1.0f / r);
      sp[i].push_back(10.0f / 3.6f);
    }
    sp[i].back() = 0.0f;
  }
  const float KP = 1.0f;
  {
    std::vector<State> fleet(n, State(-0.0f, -0.0f, 0.0f, 0.0f));
    std::vector<int> ind(n, 0);
    Vec_f pe(n, 0.0f), pth_e(n, 0.0f), ai(n);
    for (int tick = 0; tick < 100; ++tick) {
      Vec_f delta = lqr_steer_control::lqr_steering_control(fleet, cx, cy, cyaw, ck, ind, pe, pth_e);
      for (int i = 0; i < n; ++i) ai[i] = KP * (sp[i][ind[i]] - fleet[i].v);
      lqr_steer_control::update(fleet, ai, delta);
    }
    std::printf("lqr_steer_control %.6f %.6f / %.6f %.6f\n", fleet[0].x, fleet[0].y, fleet[n - 1].x, fleet[n - 1].y);
  }
  {
    std::vector<State> fleet(n, State(-0.0f, -0.0f, 0.0f, 0.0f));
    Vec_f pe(n, 0.0f), pth_e(n, 0.0f), ai(n), di(n);
    for (int tick = 0; tick < 100; ++tick) {
      std::vector<Vec_f> u = lqr_speed_steer_control::lqr_steering_control(fleet, cx, cy, cyaw, ck, sp, pe, pth_e);
      for (int i = 0; i < n; ++i) { ai[i] = u[i][0]; di[i] = u[i][1]; }
      lqr_speed_steer_control::update(fleet, ai, di);
    }
    std::printf("lqr_speed_steer_control %.6f %.6f / %.6f %.6f\n", fleet[0].x, fleet[0].y, fleet[n - 1].x,
                fleet[n - 1].y);
  }
  return 0;
}
