// reference_api.hpp — host C++ with the reference's own names, argument order and value semantics,
// on top of the C ABI (crb.h).  A CppRobotics main() re-targets to the H100 engine by including this
// header instead of <Eigen/Eigen> for the hot functions and linking libcrb.so.
//
//   ekf_estimation(xEst, PEst, z, u, Q, R)        src/extended_kalman_filter.cpp:64-78
//   pf_localization(px, pw, xEst, PEst, z, u, Rsim, Q, gen, gaussian_d)   src/particle_filter.cpp:73-109
//   mpc_solve(x0, traj_ref)                       src/model_predictive_control.cpp:255-346
//   update(state, a, delta)                       src/model_predictive_control.cpp:69-81
//   calc_ref_trajectory(...)                      src/model_predictive_control.cpp:130-170
//   resampling(px, pw, gen, uni_d)                src/particle_filter.cpp:120-148
//   solve_DARE / dlqr (4x4 and 5x5)               src/lqr_steer_control.cpp:75-96, lqr_speed_steer_control.cpp:85-106
//   dwa_control(x, u, config, goal, ob), motion(x, u, dt)   src/dynamic_window_approach.cpp:148-155, :43-50
//   MotionModel, TrajectoryOptimizer::optimizer_traj(...)    include/motion_model.h, include/trajectory_optimizer.h
//
// Eigen is not a dependency: crb::Mat<R,C> is a POD with the memory layout of
// Eigen::Matrix<float,R,C> (column-major, contiguous, no padding), enough of its interface for the
// call sites above.  Errors: the reference reports none; these shims throw std::runtime_error with
// crb_last_error_string() (e.g. when no H100 is present: there is no CPU fallback).
//
// These are single-agent calls (n = 1, or NP particles) through the *_host entry points: they exist for
// drop-in compatibility and for tests; throughput comes from calling the batched C ABI directly.
#ifndef CRB_REFERENCE_API_HPP_
#define CRB_REFERENCE_API_HPP_

#include <array>
#include <cmath>
#include <cstring>
#include <random>
#include <stdexcept>
#include <string>
#include <vector>

#include "../crb.h"

namespace crb {

template <int R, int C = 1>
struct Mat {
  float d[R * C];
  float& operator()(int r, int c = 0) { return d[r + R * c]; }
  const float& operator()(int r, int c = 0) const { return d[r + R * c]; }
  float* data() { return d; }
  const float* data() const { return d; }
  static constexpr int rows() { return R; }
  static constexpr int cols() { return C; }
  static Mat Zero() {
    Mat m;
    for (int i = 0; i < R * C; ++i) m.d[i] = 0.0f;
    return m;
  }
  static Mat Identity() {
    Mat m = Zero();
    for (int i = 0; i < (R < C ? R : C); ++i) m(i, i) = 1.0f;
    return m;
  }
};
using Vector2f = Mat<2, 1>;
using Vector4f = Mat<4, 1>;
using Matrix2f = Mat<2, 2>;
using Matrix4f = Mat<4, 4>;
using RowVector3f = Mat<1, 3>;
template <int T>
using M_XREF = Mat<4, T>;  // Eigen::Matrix<float, NX, T>, src/model_predictive_control.cpp:52

inline void check(int rc, const char* what) {
  if (rc != CRB_OK)
    throw std::runtime_error(std::string(what) + " failed (" + std::to_string(rc) +
                             "): " + crb_last_error_string());
}

// One lazily created context per thread (a crb_ctx is not thread-safe).  The session also owns a grow-only
// device arena: the shims below carve their per-call device buffers out of it, so a reference main() that
// calls update() / calc_ref_trajectory() every step does not pay cudaMalloc + cudaFree per call, and an
// exception thrown between "allocate" and "free" cannot leak device memory (there is nothing to free).
class Session {
 public:
  static crb_ctx* get() { return self().ctx_; }
  // at least n_floats floats of device memory, valid until the next scratch() call on this thread
  static float* scratch(size_t n_floats) {
    Session& s = self();
    if (n_floats > s.cap_) {
      if (s.arena_) crb_device_free(s.ctx_, s.arena_);
      s.arena_ = nullptr;
      s.cap_ = 0;
      size_t want = n_floats < 4096 ? 4096 : n_floats;
      check(crb_device_alloc(s.ctx_, &s.arena_, want * sizeof(float)), "crb_device_alloc");
      s.cap_ = want;
    }
    return (float*)s.arena_;
  }
  Session(const Session&) = delete;

 private:
  static Session& self() {
    thread_local Session s;
    return s;
  }
  Session() { check(crb_init(&ctx_, -1), "crb_init"); }
  ~Session() {
    if (arena_) crb_device_free(ctx_, arena_);
    crb_destroy(ctx_);
  }
  crb_ctx* ctx_ = nullptr;
  void* arena_ = nullptr;
  size_t cap_ = 0;
};

}  // namespace crb

namespace cpprobotics {
// include/cpprobotics_types.h:19-21
using Vec_f = std::vector<float>;
using Poi_f = std::array<float, 2>;
using Vec_Poi = std::vector<Poi_f>;
// include/motion_model.h:31-42 (same members, same constructor, no default constructor)
struct State {
  float x;
  float y;
  float yaw;
  float v;
  State(float x_, float y_, float yaw_, float v_) : x(x_), y(y_), yaw(yaw_), v(v_) {}
};
}  // namespace cpprobotics

// ---------------------------------------------------------------------------------------------------
// Reference-signature functions (global namespace, like the reference's free functions).
// ---------------------------------------------------------------------------------------------------

// src/extended_kalman_filter.cpp:64-78.  Q and R are passed through (the reference's DT stays 0.1).
inline void ekf_estimation(crb::Vector4f& xEst, crb::Matrix4f& PEst, crb::Vector2f z,
                           crb::Vector2f u, crb::Matrix4f Q, crb::Matrix2f R) {
  crb_ekf_params prm;
  crb_ekf_default_params(&prm);
  std::memcpy(prm.Q, Q.data(), sizeof(prm.Q));
  std::memcpy(prm.R, R.data(), sizeof(prm.R));
  // n = 1: SoA and AoS coincide, the Eigen column-major buffers are passed as they are
  crb::check(crb_ekf_step_batched_host(crb::Session::get(), 1, xEst.data(), PEst.data(), z.data(),
                                       u.data(), &prm, 1),
             "crb_ekf_step_batched_host");
}

// src/model_predictive_control.cpp:69-81
inline void update(cpprobotics::State& state, float a, float delta) {
  crb_ctx* ctx = crb::Session::get();
  float st[4] = {state.x, state.y, state.yaw, state.v}, u0[2] = {a, delta};
  float* dst = crb::Session::scratch(6);
  float* du = dst + 4;
  crb::check(crb_memcpy_h2d(ctx, dst, st, sizeof(st)), "crb_memcpy_h2d");
  crb::check(crb_memcpy_h2d(ctx, du, u0, sizeof(u0)), "crb_memcpy_h2d");
  crb_mpc_params prm;
  crb_mpc_default_params(&prm);
  crb::check(crb_mpc_plant_update_batched(ctx, 1, dst, du, &prm), "crb_mpc_plant_update_batched");
  crb::check(crb_memcpy_d2h(ctx, st, dst, sizeof(st)), "crb_memcpy_d2h");
  state.x = st[0]; state.y = st[1]; state.yaw = st[2]; state.v = st[3];
}

// src/model_predictive_control.cpp:255-346.  Returns the reference's vector
// [x(T) | y(T) | yaw(T) | v(T) | delta(T-1) | a(T-1)] (:54-60, :341-345); the caller reads
// output[a_start] and output[delta_start] (:376).
template <int T>
inline cpprobotics::Vec_f mpc_solve(cpprobotics::State x0, crb::M_XREF<T> traj_ref,
                                    const crb_mpc_params* params = nullptr,
                                    int32_t* status_out = nullptr) {
  static_assert(T >= 2 && T <= CRB_MPC_MAX_T, "horizon out of range");
  crb_mpc_params prm;
  if (params) prm = *params; else crb_mpc_default_params(&prm);
  const float x[4] = {x0.x, x0.y, x0.yaw, x0.v};
  cpprobotics::Vec_f result(4 * T + 2 * (T - 1));
  int32_t status = 0;
  // M_XREF is column-major 4 x T: element (k, t) at k + 4t, which is exactly field 4t + k for n = 1
  crb::check(crb_mpc_solve_batched_host(crb::Session::get(), 1, T, x, traj_ref.data(), nullptr, &prm,
                                        result.data(), nullptr, nullptr, &status, nullptr),
             "crb_mpc_solve_batched_host");
  if (status_out) *status_out = status;
  return result;
}

// src/model_predictive_control.cpp:130-170 (calc_nearest_index :107-127 inside).  ck is accepted and
// ignored like in the reference.
template <int T>
inline void calc_ref_trajectory(cpprobotics::State state, cpprobotics::Vec_f cx,
                                cpprobotics::Vec_f cy, cpprobotics::Vec_f cyaw,
                                cpprobotics::Vec_f /*ck*/, cpprobotics::Vec_f sp, float dl,
                                int& target_ind, crb::M_XREF<T>& xref) {
  crb_ctx* ctx = crb::Session::get();
  const size_t nc = cx.size();
  const float st[4] = {state.x, state.y, state.yaw, state.v};
  int32_t ti = target_ind;
  float* dc = crb::Session::scratch(4 * nc + 4 + 4 + 4 * T);   // course | state | target_ind | xref
  float* dst = dc + 4 * nc;
  float* dti = dst + 4;
  float* dxr = dti + 4;
  crb::check(crb_memcpy_h2d(ctx, dc, cx.data(), nc * sizeof(float)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, dc + nc, cy.data(), nc * sizeof(float)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, dc + 2 * nc, cyaw.data(), nc * sizeof(float)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, dc + 3 * nc, sp.data(), nc * sizeof(float)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, dst, st, sizeof(st)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, dti, &ti, sizeof(ti)), "h2d");
  crb_mpc_params prm;
  crb_mpc_default_params(&prm);
  crb::check(crb_mpc_calc_ref_trajectory_batched(ctx, 1, T, dst, dc, dc + nc, dc + 2 * nc, dc + 3 * nc,
                                                 (int32_t)nc, dl, (int32_t*)dti, dxr, &prm),
             "crb_mpc_calc_ref_trajectory_batched");
  crb::check(crb_memcpy_d2h(ctx, xref.data(), dxr, 4 * T * sizeof(float)), "d2h");
  crb::check(crb_memcpy_d2h(ctx, &ti, dti, sizeof(ti)), "d2h");
  target_ind = ti;
}

// src/particle_filter.cpp:73-109.  NP is a template parameter (a macro in the reference, :21).
// gen and gaussian_d are taken BY VALUE exactly like the reference (:78), so the caller's generator is
// not advanced; the draws are made here on the host in the reference's order (two per particle,
// :87-88) and handed to the kernel as its explicit noise input.
template <int NP>
inline void pf_localization(crb::Mat<4, NP>& px, crb::Mat<NP, 1>& pw, crb::Vector4f& xEst,
                            crb::Matrix4f& PEst, std::vector<crb::RowVector3f> z, crb::Vector2f u,
                            crb::Matrix2f Rsim, float Q, std::mt19937 gen,
                            std::normal_distribution<> gaussian_d) {
  crb_ctx* ctx = crb::Session::get();
  crb_pf_params prm;
  crb_pf_default_params(&prm);
  prm.Q = Q;
  prm.rsim_diag[0] = Rsim(0, 0);
  prm.rsim_diag[1] = Rsim(1, 1);
  prm.u[0] = u(0);
  prm.u[1] = u(1);
  // Eigen's px is 4 x NP column-major = AoS per particle; the engine wants SoA [4][NP]
  std::vector<float> sx(4 * NP), noise(2 * NP), lm(3 * z.size());
  for (int ip = 0; ip < NP; ++ip) {
    for (int k = 0; k < 4; ++k) sx[k * NP + ip] = px(k, ip);
    noise[ip] = (float)gaussian_d(gen);
    noise[NP + ip] = (float)gaussian_d(gen);
  }
  for (size_t i = 0; i < z.size(); ++i)
    for (int k = 0; k < 3; ++k) lm[3 * i + k] = z[i](0, k);
  float* dpx = crb::Session::scratch(7 * (size_t)NP);   // px [4][NP] | pw [NP] | noise [2][NP]
  float* dpw = dpx + 4 * NP;
  float* dn = dpw + NP;
  crb::check(crb_memcpy_h2d(ctx, dpx, sx.data(), sx.size() * sizeof(float)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, dpw, pw.data(), NP * sizeof(float)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, dn, noise.data(), noise.size() * sizeof(float)), "h2d");
  crb::check(crb_pf_predict_weight_batched(ctx, NP, dpx, dpw, dn, 0, lm.data(), (int)z.size(), &prm),
             "crb_pf_predict_weight_batched");                          // :81-102
  crb::check(crb_pf_estimate(ctx, NP, dpx, dpw, xEst.data(), PEst.data(), nullptr),
             "crb_pf_estimate");                                        // :104-107
  crb::check(crb_memcpy_d2h(ctx, sx.data(), dpx, sx.size() * sizeof(float)), "d2h");
  crb::check(crb_memcpy_d2h(ctx, pw.data(), dpw, NP * sizeof(float)), "d2h");
  for (int ip = 0; ip < NP; ++ip)
    for (int k = 0; k < 4; ++k) px(k, ip) = sx[k * NP + ip];
}

// src/particle_filter.cpp:120-148.  gen and uni_d BY VALUE like the reference (:122-123: the caller's
// generator is not advanced, so every call sees the same draws - the reference's quirk).  The NP draws
// are made here in the reference's order (one per particle, :133) and handed to the engine as its
// explicit uniforms; NTh = NP/2 (:22).  Deviations (documented in crb.h): the cumulative weights are
// accumulated in double, the draw is narrowed to float before use.
template <int NP>
inline void resampling(crb::Mat<4, NP>& px, crb::Mat<NP, 1>& pw, std::mt19937 gen,
                       std::uniform_real_distribution<> uni_d) {
  crb_ctx* ctx = crb::Session::get();
  std::vector<float> sx(4 * NP), un(NP);
  for (int ip = 0; ip < NP; ++ip) {
    for (int k = 0; k < 4; ++k) sx[k * NP + ip] = px(k, ip);
    un[ip] = (float)uni_d(gen);
  }
  float* dpx = crb::Session::scratch(10 * (size_t)NP);   // px [4][NP] | px_tmp [4][NP] | pw [NP] | uniforms [NP]
  float* dtmp = dpx + 4 * NP;
  float* dpw = dtmp + 4 * NP;
  float* du = dpw + NP;
  crb::check(crb_memcpy_h2d(ctx, dpx, sx.data(), sx.size() * sizeof(float)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, dpw, pw.data(), NP * sizeof(float)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, du, un.data(), NP * sizeof(float)), "h2d");
  int did = 0;
  // NTh = NP / 2 is an INTEGER expression in the reference (:22)
  crb::check(crb_pf_resample(ctx, NP, dpx, dpw, dtmp, du, 0, (float)(NP / 2), &did, nullptr),
             "crb_pf_resample");
  if (did) {
    crb::check(crb_memcpy_d2h(ctx, sx.data(), dpx, sx.size() * sizeof(float)), "d2h");
    crb::check(crb_memcpy_d2h(ctx, pw.data(), dpw, NP * sizeof(float)), "d2h");
    for (int ip = 0; ip < NP; ++ip)
      for (int k = 0; k < 4; ++k) px(k, ip) = sx[k * NP + ip];
  }
}

// solve_DARE + dlqr: src/lqr_steer_control.cpp:75-96 (nx = 4, scalar R) and
// src/lqr_speed_steer_control.cpp:85-106 (nx = 5, 2x2 R).  One problem per call through the batched entry.
namespace crb {
using Matrix5f = Mat<5, 5>;
using Matrix52f = Mat<5, 2>;
using Matrix25f = Mat<2, 5>;
using RowVector4f = Mat<1, 4>;

template <int NX, int NU>
inline void dlqr_impl(const float* A, const float* B, const float* Q, const float* R, float* K, float* X) {
  crb_ctx* ctx = Session::get();
  const size_t na = NX * NX, nb = NX * NU, nr = NU * NU, nk = NU * NX;
  float* dA = Session::scratch(2 * na + nb + nr + nk + na);
  float *dB = dA + na, *dQ = dB + nb, *dR = dQ + na, *dK = dR + nr, *dX = dK + nk;
  check(crb_memcpy_h2d(ctx, dA, A, na * sizeof(float)), "h2d");
  check(crb_memcpy_h2d(ctx, dB, B, nb * sizeof(float)), "h2d");
  check(crb_memcpy_h2d(ctx, dQ, Q, na * sizeof(float)), "h2d");
  check(crb_memcpy_h2d(ctx, dR, R, nr * sizeof(float)), "h2d");
  check(crb_lqr_dlqr_batched(ctx, 1, NX, NU, dA, dB, dQ, dR, /*maxiter :77*/ 150, /*eps :78*/ 0.01f, dK, dX,
                             nullptr),
        "crb_lqr_dlqr_batched");
  if (K) check(crb_memcpy_d2h(ctx, K, dK, nk * sizeof(float)), "d2h");
  if (X) check(crb_memcpy_d2h(ctx, X, dX, na * sizeof(float)), "d2h");
}
}  // namespace crb

inline crb::Matrix4f solve_DARE(crb::Matrix4f A, crb::Vector4f B, crb::Matrix4f Q, float R) {
  crb::Matrix4f X;
  crb::dlqr_impl<4, 1>(A.data(), B.data(), Q.data(), &R, nullptr, X.data());
  return X;
}
inline crb::RowVector4f dlqr(crb::Matrix4f A, crb::Vector4f B, crb::Matrix4f Q, float R) {
  crb::RowVector4f K;
  crb::dlqr_impl<4, 1>(A.data(), B.data(), Q.data(), &R, K.data(), nullptr);
  return K;
}
inline crb::Matrix5f solve_DARE(crb::Matrix5f A, crb::Matrix52f B, crb::Matrix5f Q, crb::Matrix2f R) {
  crb::Matrix5f X;
  crb::dlqr_impl<5, 2>(A.data(), B.data(), Q.data(), R.data(), nullptr, X.data());
  return X;
}
inline crb::Matrix25f dlqr(crb::Matrix5f A, crb::Matrix52f B, crb::Matrix5f Q, crb::Matrix2f R) {
  crb::Matrix25f K;
  crb::dlqr_impl<5, 2>(A.data(), B.data(), Q.data(), R.data(), K.data(), nullptr);
  return K;
}

// src/dynamic_window_approach.cpp.  Its State, Control, Point, Traj and Obstacle (:18-23) are aliases of exactly
// these std types, and its Config (:25-41) is the program's own class, read here by member name.
namespace crb {
template <class Config>
inline crb_dwa_params dwa_params_of(const Config& c) {
  crb_dwa_params p;
  p.max_speed = c.max_speed; p.min_speed = c.min_speed; p.max_yawrate = c.max_yawrate;
  p.max_accel = c.max_accel; p.robot_radius = c.robot_radius; p.max_dyawrate = c.max_dyawrate;
  p.v_reso = c.v_reso; p.yawrate_reso = c.yawrate_reso; p.dt = c.dt; p.predict_time = c.predict_time;
  p.to_goal_cost_gain = c.to_goal_cost_gain; p.speed_cost_gain = c.speed_cost_gain;
  return p;
}
}  // namespace crb

// dwa_control :148-155: sets u and returns the chosen rollout (empty when no sample is admissible, like the
// reference).  ob must have at most CRB_DWA_MAX_OBSTACLES rows.
template <class Config>
inline std::vector<std::array<float, 5>> dwa_control(std::array<float, 5> x, std::array<float, 2>& u, Config config,
                                                     std::array<float, 2> goal,
                                                     std::vector<std::array<float, 2>> ob) {
  crb_ctx* ctx = crb::Session::get();
  const crb_dwa_params prm = crb::dwa_params_of(config);
  int n_pts = 0;
  crb::check(crb_dwa_rollout_points(&prm, &n_pts), "crb_dwa_rollout_points");
  const size_t n_ob = ob.size();
  // x [5] | u [2] | goal [2] | ob [n_ob][2] | best [1] | traj [5 n_pts]  (n = 1: SoA and AoS coincide)
  float* dx = crb::Session::scratch(10 + 2 * n_ob + 5 * (size_t)n_pts);
  float *du = dx + 5, *dg = du + 2, *dob = dg + 2, *dbest = dob + 2 * n_ob, *dtraj = dbest + 1;
  crb::check(crb_memcpy_h2d(ctx, dx, x.data(), 5 * sizeof(float)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, du, u.data(), 2 * sizeof(float)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, dg, goal.data(), 2 * sizeof(float)), "h2d");
  if (n_ob) crb::check(crb_memcpy_h2d(ctx, dob, ob.data(), 2 * n_ob * sizeof(float)), "h2d");
  crb::check(crb_dwa_control_batched(ctx, 1, dx, du, dg, dob, (int)n_ob, &prm, nullptr, (int32_t*)dbest, dtraj),
             "crb_dwa_control_batched");
  int32_t best = -1;
  std::vector<std::array<float, 5>> traj((size_t)n_pts);
  crb::check(crb_memcpy_d2h(ctx, u.data(), du, 2 * sizeof(float)), "d2h");
  crb::check(crb_memcpy_d2h(ctx, &best, dbest, sizeof(best)), "d2h");
  crb::check(crb_memcpy_d2h(ctx, traj.data(), dtraj, 5 * (size_t)n_pts * sizeof(float)), "d2h");
  if (best < 0) traj.clear();
  return traj;
}

// motion :43-50 (the plant step of main() :194)
inline std::array<float, 5> motion(std::array<float, 5> x, std::array<float, 2> u, float dt) {
  crb_ctx* ctx = crb::Session::get();
  float* dx = crb::Session::scratch(7);
  crb::check(crb_memcpy_h2d(ctx, dx, x.data(), 5 * sizeof(float)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, dx + 5, u.data(), 2 * sizeof(float)), "h2d");
  crb::check(crb_dwa_motion_batched(ctx, 1, dx, dx + 5, dt), "crb_dwa_motion_batched");
  crb::check(crb_memcpy_d2h(ctx, x.data(), dx, 5 * sizeof(float)), "d2h");
  return x;
}

// include/motion_model.h:22-92 and include/trajectory_optimizer.h:32-51: the same types, members and constructors.
// MotionModel's trajectories and TrajectoryOptimizer::optimizer_traj run through the batched entry points with
// n = 1.  The optimizer's drawing (visualize, save) and its console message on convergence are not reproduced.
namespace cpprobotics {
struct Parameter {
  float distance;
  std::array<float, 3> steering_sequence{{0, 0, 0}};
  Parameter(float distance_, std::array<float, 3> steering_sequence_)
      : distance(distance_), steering_sequence(steering_sequence_) {}
};
struct TrajState {
  float x;
  float y;
  float yaw;
  TrajState(float x_, float y_, float yaw_) : x(x_), y(y_), yaw(yaw_) {}
};
using Traj = std::vector<TrajState>;

namespace detail {
// state [4] | target [3] | param [4] | len, status, iters | last [3] | traj [3 max_pts]  (n = 1: SoA is AoS)
inline float* mptg_scratch(int max_pts) { return crb::Session::scratch(17 + 3 * (size_t)max_pts); }
inline Traj mptg_read_traj(crb_ctx* ctx, const float* dtraj, int len) {
  std::vector<float> buf(3 * (size_t)len);
  if (len) crb::check(crb_memcpy_d2h(ctx, buf.data(), dtraj, buf.size() * sizeof(float)), "d2h");
  Traj t;
  t.reserve((size_t)len);
  for (int k = 0; k < len; ++k) t.push_back(TrajState(buf[3 * k], buf[3 * k + 1], buf[3 * k + 2]));
  return t;
}
}  // namespace detail

class MotionModel {
 public:
  const float base_l;
  const float ds;
  State state;
  MotionModel(float base_l_, float ds_, State state_) : base_l(base_l_), ds(ds_), state(state_) {}
  // generate_trajectory :110-131
  Traj generate_trajectory(Parameter p) const {
    int len = 0;
    float last[3];
    return run(p, 256, &len, last, true);
  }
  // generate_last_state :133-150
  TrajState generate_last_state(Parameter p) const {
    int len = 0;
    float last[3];
    run(p, 0, &len, last, false);
    return TrajState(last[0], last[1], last[2]);
  }
  crb_mptg_params params() const {
    crb_mptg_params prm;
    crb_mptg_default_params(&prm);
    prm.base_l = base_l;
    prm.ds = ds;
    return prm;
  }

 private:
  Traj run(const Parameter& p, int max_pts, int* len, float* last, bool want_traj) const {
    crb_ctx* ctx = crb::Session::get();
    const crb_mptg_params prm = params();
    for (;;) {
      float* d = detail::mptg_scratch(max_pts);
      const float st[4] = {state.x, state.y, state.yaw, state.v};
      const float q[4] = {p.distance, p.steering_sequence[0], p.steering_sequence[1], p.steering_sequence[2]};
      crb::check(crb_memcpy_h2d(ctx, d, st, sizeof(st)), "h2d");
      crb::check(crb_memcpy_h2d(ctx, d + 7, q, sizeof(q)), "h2d");
      crb::check(crb_mptg_generate_trajectory_batched(ctx, 1, d, d + 7, &prm, max_pts, want_traj ? d + 17 : nullptr,
                                                      (int32_t*)(d + 11), d + 14, (int32_t*)(d + 12)),
                 "crb_mptg_generate_trajectory_batched");
      int32_t ls[2];
      crb::check(crb_memcpy_d2h(ctx, ls, d + 11, sizeof(ls)), "d2h");
      crb::check(crb_memcpy_d2h(ctx, last, d + 14, 3 * sizeof(float)), "d2h");
      if (ls[1] != CRB_MPTG_CONVERGED)
        throw std::runtime_error("generate_trajectory: the roll-out stopped with status " + std::to_string(ls[1]));
      *len = ls[0];
      if (!want_traj) return Traj();
      if (ls[0] <= max_pts) return detail::mptg_read_traj(ctx, d + 17, ls[0]);
      max_pts = ls[0];
    }
  }
};

class TrajectoryOptimizer {
 public:
  MotionModel m_model;
  Parameter p;
  TrajState target;
  TrajectoryOptimizer(MotionModel m_model_, Parameter init_p_, TrajState target_)
      : m_model(m_model_), p(init_p_), target(target_) {}
  // optimizer_traj :53-128: updates p and returns the last nominal trajectory.  A problem the reference leaves
  // undefined, or that is outside the exact range of the restated libm (crb.h, CRB_MPTG_*), throws.
  Traj optimizer_traj(int max_iter, float cost_th, std::vector<float> h_step, bool visualize = false,
                      bool save = false) {
    (void)visualize;
    (void)save;
    if (h_step.size() < 3) throw std::runtime_error("optimizer_traj: h_step needs 3 entries");
    crb_ctx* ctx = crb::Session::get();
    crb_mptg_params prm = m_model.params();
    prm.max_iter = max_iter;
    prm.cost_th = cost_th;
    for (int k = 0; k < 3; ++k) prm.h_step[k] = h_step[k];
    int max_pts = 256;
    for (;;) {
      float* d = detail::mptg_scratch(max_pts);
      const float st[4] = {m_model.state.x, m_model.state.y, m_model.state.yaw, m_model.state.v};
      const float tg[3] = {target.x, target.y, target.yaw};
      const float q[4] = {p.distance, p.steering_sequence[0], p.steering_sequence[1], p.steering_sequence[2]};
      crb::check(crb_memcpy_h2d(ctx, d, st, sizeof(st)), "h2d");
      crb::check(crb_memcpy_h2d(ctx, d + 4, tg, sizeof(tg)), "h2d");
      crb::check(crb_memcpy_h2d(ctx, d + 7, q, sizeof(q)), "h2d");
      crb::check(crb_mptg_optimize_batched(ctx, 1, d, d + 4, d + 7, &prm, max_pts, d + 17, (int32_t*)(d + 11),
                                           nullptr, (int32_t*)(d + 12), (int32_t*)(d + 13)),
                 "crb_mptg_optimize_batched");
      int32_t ls[2];
      crb::check(crb_memcpy_d2h(ctx, ls, d + 11, sizeof(ls)), "d2h");
      if (ls[1] != CRB_MPTG_CONVERGED && ls[1] != CRB_MPTG_MAX_ITER_REACHED)
        throw std::runtime_error("optimizer_traj: stopped with status " + std::to_string(ls[1]));
      if (ls[0] > max_pts) {  // the same problem again with room for the whole trajectory
        max_pts = ls[0];
        continue;
      }
      float qo[4];
      crb::check(crb_memcpy_d2h(ctx, qo, d + 7, sizeof(qo)), "d2h");
      p.distance = qo[0];
      for (int k = 0; k < 3; ++k) p.steering_sequence[k] = qo[k + 1];
      return detail::mptg_read_traj(ctx, d + 17, ls[0]);
    }
  }
};
}  // namespace cpprobotics

#endif  // CRB_REFERENCE_API_HPP_
