// oracle/shim/ref_wrap_dwa.cpp — C entry points around the reference's own src/dynamic_window_approach.cpp.  The
// file is #included from where it lies (REF_SRC, set by oracle/dwa.mk) with main() renamed; nothing of it is copied
// into this repository.  <algorithm> and <limits> come first: the file uses std::max / std::min and
// std::numeric_limits and relies on real OpenCV's headers to include them.
#include <algorithm>
#include <limits>

#define main crb_reference_main
#include REF_SRC
#undef main

extern "C" {
// Config :25-41 set member by member from cfg[12] (crb_dwa_params order)
static Config ref_config(const float* cfg) {
  Config c;
  c.max_speed = cfg[0]; c.min_speed = cfg[1]; c.max_yawrate = cfg[2]; c.max_accel = cfg[3];
  c.robot_radius = cfg[4]; c.max_dyawrate = cfg[5]; c.v_reso = cfg[6]; c.yawrate_reso = cfg[7];
  c.dt = cfg[8]; c.predict_time = cfg[9]; c.to_goal_cost_gain = cfg[10]; c.speed_cost_gain = cfg[11];
  return c;
}
// Config's own initialisers, for the test that the library's defaults are the reference's
void ref_dwa_default_config(float* cfg) {
  Config c;
  const float v[12] = {c.max_speed, c.min_speed, c.max_yawrate, c.max_accel, c.robot_radius, c.max_dyawrate,
                       c.v_reso, c.yawrate_reso, c.dt, c.predict_time, c.to_goal_cost_gain, c.speed_cost_gain};
  for (int i = 0; i < 12; ++i) cfg[i] = v[i];
}
// dwa_control :148-155 for one robot.  u in/out; traj gets the returned Traj (5 floats per point) and
// *n_pts its size (0 when it is empty).  *cost is final_cost of the returned trajectory evaluated with the
// reference's own cost functions (:131-134), or min_cost's initial 10000 when nothing was admissible.
void ref_dwa_control(const float* x, float* u, const float* goal, const float* ob, int n_ob, const float* cfg,
                     float* traj, int* n_pts, float* cost) {
  Config c = ref_config(cfg);
  State xs = {{x[0], x[1], x[2], x[3], x[4]}};
  Control us = {{u[0], u[1]}};
  Point g = {{goal[0], goal[1]}};
  Obstacle o;
  for (int k = 0; k < n_ob; ++k) o.push_back(Point{{ob[2 * k], ob[2 * k + 1]}});
  Traj t = dwa_control(xs, us, c, g, o);
  u[0] = us[0]; u[1] = us[1];
  *n_pts = (int)t.size();
  for (size_t k = 0; k < t.size(); ++k)
    for (int j = 0; j < 5; ++j) traj[5 * k + j] = t[k][j];
  *cost = t.empty() ? 10000.0f
                    : calc_to_goal_cost(t, g, c) + c.speed_cost_gain * (c.max_speed - t.back()[3]) +
                          calc_obstacle_cost(t, o, c);
}
void ref_dwa_motion(const float* x, const float* u, float dt, float* out) {
  State s = motion(State{{x[0], x[1], x[2], x[3], x[4]}}, Control{{u[0], u[1]}}, dt);
  for (int j = 0; j < 5; ++j) out[j] = s[j];
}
}
