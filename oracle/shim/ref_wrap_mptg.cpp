// oracle/shim/ref_wrap_mptg.cpp — C entry points around the reference's own include/trajectory_optimizer.h (and the
// include/motion_model.h it includes).  The header is #included from where it lies (REF_HDR, set by oracle/Makefile);
// nothing of it is copied into this repository.  <limits> comes first: the header uses std::numeric_limits and
// relies on real OpenCV's headers to include it.
#include <limits>

#include REF_HDR

using namespace cpprobotics;

namespace {
// the cost of :108-109 for a returned trajectory's last point (calc_diff :130-135 is private: restated with the
// header's own YAW_P2P)
float last_cost(const TrajState& t, const TrajState& target) {
  const float dx = target.x - t.x, dy = target.y - t.y, yaw_ = target.yaw - t.yaw;
  const float dyaw = YAW_P2P(yaw_);
  return std::sqrt(std::pow(dx, 2) + std::pow(dy, 2) + std::pow(dyaw, 2));
}
}  // namespace

extern "C" {
// optimizer_traj(max_iter, cost_th, h) for one problem.  st[4] = (x, y, yaw, v), tg[3], p[4] in/out = (distance,
// steering_sequence[0..2]) as the optimizer left it, traj[3 * max_pts] and *len = the returned Traj (its full
// size; at most max_pts points copied), *cost = the cost of its last point (NaN when it is empty).
void ref_mptg_optimize(const float* st, const float* tg, float* p, float base_l, float ds, int max_iter,
                       float cost_th, const float* h, float* traj, int max_pts, int* len, float* cost) {
  MotionModel m(base_l, ds, State(st[0], st[1], st[2], st[3]));
  TrajState target(tg[0], tg[1], tg[2]);
  TrajectoryOptimizer opt(m, Parameter(p[0], {{p[1], p[2], p[3]}}), target);
  Traj t = opt.optimizer_traj(max_iter, cost_th, std::vector<float>{h[0], h[1], h[2]});
  p[0] = opt.p.distance;
  for (int k = 0; k < 3; ++k) p[k + 1] = opt.p.steering_sequence[k];
  *len = (int)t.size();
  for (size_t k = 0; k < t.size() && (int)k < max_pts; ++k) {
    traj[3 * k] = t[k].x;
    traj[3 * k + 1] = t[k].y;
    traj[3 * k + 2] = t[k].yaw;
  }
  *cost = t.empty() ? std::numeric_limits<float>::quiet_NaN() : last_cost(t.back(), target);
}
// MotionModel::generate_trajectory and generate_last_state for one parameter
void ref_mptg_generate(const float* st, const float* p, float base_l, float ds, float* traj, int max_pts, int* len,
                       float* last) {
  MotionModel m(base_l, ds, State(st[0], st[1], st[2], st[3]));
  Parameter q(p[0], {{p[1], p[2], p[3]}});
  Traj t = m.generate_trajectory(q);
  *len = (int)t.size();
  for (size_t k = 0; k < t.size() && (int)k < max_pts; ++k) {
    traj[3 * k] = t[k].x;
    traj[3 * k + 1] = t[k].y;
    traj[3 * k + 2] = t[k].yaw;
  }
  TrajState l = m.generate_last_state(q);
  last[0] = l.x;
  last[1] = l.y;
  last[2] = l.yaw;
}
}
