// reference_api.hpp — host C++ with the reference's own names, argument order and value semantics,
// on top of the C ABI (crb.h).  A CppRobotics main() re-targets to the H100 engine by including this
// header instead of <Eigen/Eigen> for the hot functions and linking libcrb.so.
//
//   ekf_estimation(xEst, PEst, z, u, Q, R)        src/extended_kalman_filter.cpp:64-78 (also over vectors of robots)
//   pf_localization(px, pw, xEst, PEst, z, u, Rsim, Q, gen, gaussian_d)   src/particle_filter.cpp:73-109
//   mpc_solve(x0, traj_ref)                       src/model_predictive_control.cpp:255-346
//   update(state, a, delta)                       src/model_predictive_control.cpp:69-81
//   calc_ref_trajectory(...)                      src/model_predictive_control.cpp:130-170
//   resampling(px, pw, gen, uni_d)                src/particle_filter.cpp:120-148
//   pf_localization_resampling(px, pw, xEst, PEst, z, u, ...)   the demo's tick :270-271 for a fleet, one launch
//   solve_DARE / dlqr (4x4 and 5x5)               src/lqr_steer_control.cpp:75-96, lqr_speed_steer_control.cpp:85-106
//   dwa_control(x, u, config, goal, ob), motion(x, u, dt)   src/dynamic_window_approach.cpp:148-155, :43-50 (also over
//                                                            vectors of robots, with one Config or a Config per robot)
//   MotionModel, TrajectoryOptimizer::optimizer_traj(...)    include/motion_model.h, include/trajectory_optimizer.h
//   calc_{uniform_polar,biased_polar,lane}_states, search_nearest_one_from_lookuptable, generate_path
//                                                            src/state_lattice_planner.cpp:47-155
//   a_star_planning(sx, sy, gx, gy, ox, oy, reso, rr), dijkstra_star_planning(...)
//                                                            src/a_star.cpp:110-244, src/dijkstra.cpp
//   Node, RRT(start, end, ob_list, rand_area, expand_dis, ...).planning()   include/rrt.h:21-159
//   lqr_steer_control::{lqr_steering_control, update}        src/lqr_steer_control.cpp:98-146
//   lqr_speed_steer_control::{lqr_steering_control, update}  src/lqr_speed_steer_control.cpp:108-164
//                                                            (namespaces: ::update above is the MPC program's)
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

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <memory>
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

// ekf_estimation for a fleet, each robot with its own Q and R: robot i is ekf_estimation(xEst[i], PEst[i], z[i], u[i],
// Q[i], R[i]) with the reference's DT, all in one launch of crb_ekf_step_many_batched with one model per robot.
inline void ekf_estimation(std::vector<crb::Vector4f>& xEst, std::vector<crb::Matrix4f>& PEst,
                           const std::vector<crb::Vector2f>& z, const std::vector<crb::Vector2f>& u,
                           const std::vector<crb::Matrix4f>& Q, const std::vector<crb::Matrix2f>& R) {
  const size_t n = xEst.size();
  if (PEst.size() != n || z.size() != n || u.size() != n || Q.size() != n || R.size() != n)
    throw std::runtime_error("ekf_estimation: xEst, PEst, z, u, Q and R differ in length");
  if (n == 0) return;
  crb_ctx* ctx = crb::Session::get();
  crb_ekf_params dflt;
  crb_ekf_default_params(&dflt);
  // host and device: models [n] (22 floats each) | x [4][n] | P [16][n] | z [2][n] | u [2][n] | model_of [n]
  const size_t nm = sizeof(crb_ekf_params) / sizeof(float);
  std::vector<float> h((nm + 25) * n);
  std::vector<crb_ekf_params> models(n, dflt);
  float* hx = h.data() + nm * n;
  for (size_t i = 0; i < n; ++i) {
    std::memcpy(models[i].Q, Q[i].data(), sizeof(models[i].Q));
    std::memcpy(models[i].R, R[i].data(), sizeof(models[i].R));
    for (int f = 0; f < 4; ++f) hx[f * n + i] = xEst[i](f);
    for (int f = 0; f < 16; ++f) hx[(4 + f) * n + i] = PEst[i].data()[f];
    for (int f = 0; f < 2; ++f) hx[(20 + f) * n + i] = z[i](f);
    for (int f = 0; f < 2; ++f) hx[(22 + f) * n + i] = u[i](f);
    const int32_t m = (int32_t)i;
    std::memcpy(hx + 24 * n + i, &m, sizeof(m));
  }
  std::memcpy(h.data(), models.data(), n * sizeof(crb_ekf_params));
  float* d = crb::Session::scratch(h.size());
  float* dx = d + nm * n;
  crb::check(crb_memcpy_h2d(ctx, d, h.data(), h.size() * sizeof(float)), "crb_memcpy_h2d");
  crb::check(crb_ekf_step_many_batched(ctx, (int64_t)n, dx, dx + 4 * n, dx + 20 * n, dx + 22 * n,
                                       (const crb_ekf_params*)d, (int32_t)n, (const int32_t*)(dx + 24 * n), 1,
                                       nullptr),
             "crb_ekf_step_many_batched");
  crb::check(crb_memcpy_d2h(ctx, hx, dx, 20 * n * sizeof(float)), "crb_memcpy_d2h");
  for (size_t i = 0; i < n; ++i) {
    for (int f = 0; f < 4; ++f) xEst[i](f) = hx[f * n + i];
    for (int f = 0; f < 16; ++f) PEst[i].data()[f] = hx[(4 + f) * n + i];
  }
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

// The demo's tick for a fleet: pf_localization(px, pw, xEst, PEst, z, u, Rsim, Q, gen, gaussian_d) followed by
// resampling(px, pw, gen2, uni_d) (src/particle_filter.cpp:270-271) for every robot r, with its own particles px[r],
// weights pw[r], observations z[r] and control u[r], in ONE crb_pf_step_many_batched launch.  Each robot's generators
// are gen[r] and gen2[r], copied like the single-robot overloads take them by value (the caller's are not advanced),
// and the distributions are copied per robot, so robot r draws exactly what the two single-robot calls would: 2 NP
// normals from gen[r] (two per particle, :87-88), then NP uniforms from gen2[r] (one per particle, :133).  NTh = NP/2.
// Each robot's list holds at most CRB_PF_MAX_LANDMARKS rows.
template <int NP>
inline void pf_localization_resampling(std::vector<crb::Mat<4, NP>>& px, std::vector<crb::Mat<NP, 1>>& pw,
                                       std::vector<crb::Vector4f>& xEst, std::vector<crb::Matrix4f>& PEst,
                                       const std::vector<std::vector<crb::RowVector3f>>& z,
                                       const std::vector<crb::Vector2f>& u, crb::Matrix2f Rsim, float Q,
                                       std::vector<std::mt19937> gen, std::normal_distribution<> gaussian_d,
                                       std::vector<std::mt19937> gen2, std::uniform_real_distribution<> uni_d) {
  const size_t nr = px.size();
  if (pw.size() != nr || z.size() != nr || u.size() != nr || gen.size() != nr || gen2.size() != nr)
    throw std::runtime_error("pf_localization_resampling: px, pw, z, u, gen and gen2 need one entry per robot");
  xEst.resize(nr);
  PEst.resize(nr);
  if (nr == 0) return;
  crb_ctx* ctx = crb::Session::get();
  crb_pf_params prm;
  crb_pf_default_params(&prm);
  prm.Q = Q;
  prm.rsim_diag[0] = Rsim(0, 0);
  prm.rsim_diag[1] = Rsim(1, 1);
  const size_t n = nr * NP;
  std::vector<float> sx(4 * n), sw(n), noise(2 * n), un(n), su(2 * nr), rows;
  std::vector<int64_t> off(nr + 1, 0);
  std::vector<int32_t> of(nr);
  for (size_t r = 0; r < nr; ++r) {
    std::normal_distribution<> gd = gaussian_d;       // pf_localization's by-value arguments
    std::uniform_real_distribution<> ud = uni_d;      // resampling's
    for (int ip = 0; ip < NP; ++ip) {
      const size_t j = r * NP + ip;
      for (int k = 0; k < 4; ++k) sx[k * n + j] = px[r](k, ip);   // Eigen's 4 x NP (AoS) -> SoA [4][n]
      sw[j] = pw[r](ip);
      noise[j] = (float)gd(gen[r]);
      noise[n + j] = (float)gd(gen[r]);
    }
    for (int ip = 0; ip < NP; ++ip) un[r * NP + ip] = (float)ud(gen2[r]);
    su[r] = u[r](0);
    su[nr + r] = u[r](1);
    for (const crb::RowVector3f& zi : z[r])
      for (int k = 0; k < 3; ++k) rows.push_back(zi(0, k));
    off[r + 1] = off[r] + (int64_t)z[r].size();
    of[r] = (int32_t)r;
  }
  // device layout (floats): px | px_next | pw | noise | uniforms | u | rows | z_off (int64) | z_of | result (f64)
  const size_t nrow = rows.size();
  size_t o_off = 12 * n + 2 * nr + nrow;
  o_off += o_off & 1;                                   // 8-byte alignment for the int64 offsets
  const size_t o_of = o_off + 2 * (nr + 1);
  size_t o_res = o_of + nr;
  o_res += o_res & 1;
  float* d = crb::Session::scratch(o_res + 2 * (size_t)CRB_PF_RESULT_LEN * nr);
  float *dpx = d, *dpxn = d + 4 * n, *dpw = d + 8 * n, *dn = d + 9 * n, *dun = d + 11 * n, *du = d + 12 * n;
  float* drows = du + 2 * nr;
  int64_t* doff = (int64_t*)(d + o_off);
  int32_t* dof = (int32_t*)(d + o_of);
  double* dres = (double*)(d + o_res);
  crb::check(crb_memcpy_h2d(ctx, dpx, sx.data(), sx.size() * sizeof(float)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, dpw, sw.data(), sw.size() * sizeof(float)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, dn, noise.data(), noise.size() * sizeof(float)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, dun, un.data(), un.size() * sizeof(float)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, du, su.data(), su.size() * sizeof(float)), "h2d");
  if (nrow) crb::check(crb_memcpy_h2d(ctx, drows, rows.data(), nrow * sizeof(float)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, doff, off.data(), off.size() * sizeof(int64_t)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, dof, of.data(), of.size() * sizeof(int32_t)), "h2d");
  crb::check(crb_pf_step_many_batched(ctx, (int64_t)nr, NP, dpx, dpw, dpxn, du, dn, 0, drows, (int64_t)nrow / 3,
                                      doff, (int32_t)nr, dof, &prm, dun, 0, (float)(NP / 2), dres, nullptr),
             "crb_pf_step_many_batched");               // :73-148; NTh = NP / 2 is an integer expression (:22)
  std::vector<double> res((size_t)CRB_PF_RESULT_LEN * nr);
  crb::check(crb_memcpy_d2h(ctx, sx.data(), dpxn, sx.size() * sizeof(float)), "d2h");   // resampled or a copy
  crb::check(crb_memcpy_d2h(ctx, sw.data(), dpw, sw.size() * sizeof(float)), "d2h");
  crb::check(crb_memcpy_d2h(ctx, res.data(), dres, res.size() * sizeof(double)), "d2h");
  for (size_t r = 0; r < nr; ++r) {
    for (int ip = 0; ip < NP; ++ip) {
      for (int k = 0; k < 4; ++k) px[r](k, ip) = sx[k * n + r * NP + ip];
      pw[r](ip) = sw[r * NP + ip];
    }
    for (int k = 0; k < 4; ++k) xEst[r](k) = (float)res[k * nr + r];
    for (int k = 0; k < 16; ++k) PEst[r].d[k] = (float)res[(4 + k) * nr + r];   // column-major, like Eigen
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

// dwa_control for a fleet, each robot among its own obstacles: robot i is dwa_control(x[i], u[i], config, goal[i],
// ob[i]) (u[i] set, its rollout returned in element i, empty when no sample is admissible), all in one launch of
// crb_dwa_control_many_batched.  Each ob[i] must have at most CRB_DWA_MAX_OBSTACLES rows.
template <class Config>
inline std::vector<std::vector<std::array<float, 5>>> dwa_control(
    const std::vector<std::array<float, 5>>& x, std::vector<std::array<float, 2>>& u, Config config,
    const std::vector<std::array<float, 2>>& goal, const std::vector<std::vector<std::array<float, 2>>>& ob) {
  const size_t n = x.size();
  if (u.size() != n || goal.size() != n || ob.size() != n)
    throw std::runtime_error("dwa_control: x, u, goal and ob differ in length");
  std::vector<std::vector<std::array<float, 5>>> out(n);
  if (n == 0) return out;
  crb_ctx* ctx = crb::Session::get();
  const crb_dwa_params prm = crb::dwa_params_of(config);
  int n_pts = 0;
  crb::check(crb_dwa_rollout_points(&prm, &n_pts), "crb_dwa_rollout_points");
  // host: ob_off [n + 1] int64 | ob_of [n] int32 | x [5][n] | u [2][n] | goal [2][n] | ob [n_rows][2]
  std::vector<int64_t> off(n + 1, 0);
  for (size_t i = 0; i < n; ++i) off[i + 1] = off[i] + (int64_t)ob[i].size();
  const size_t n_rows = (size_t)off[n];
  std::vector<float> h(2 * (n + 1) + n + 9 * n + 2 * n_rows);
  std::memcpy(h.data(), off.data(), off.size() * sizeof(int64_t));
  float* hx = h.data() + 3 * n + 2;
  for (size_t i = 0; i < n; ++i) {
    const int32_t s = (int32_t)i;
    std::memcpy(h.data() + 2 * (n + 1) + i, &s, 4);
    for (int f = 0; f < 5; ++f) hx[f * n + i] = x[i][f];
    for (int f = 0; f < 2; ++f) hx[(5 + f) * n + i] = u[i][f];
    for (int f = 0; f < 2; ++f) hx[(7 + f) * n + i] = goal[i][f];
    for (size_t k = 0; k < ob[i].size(); ++k) {
      hx[9 * n + 2 * (off[i] + k)] = ob[i][k][0];
      hx[9 * n + 2 * (off[i] + k) + 1] = ob[i][k][1];
    }
  }
  // device: the host block | best [n] | traj [5 n_pts][n]; the arena comes from cudaMalloc, so ob_off is aligned
  float* d = crb::Session::scratch(h.size() + n + 5 * (size_t)n_pts * n);
  float *dx = d + 3 * n + 2, *dbest = d + h.size(), *dtraj = dbest + n;
  crb::check(crb_memcpy_h2d(ctx, d, h.data(), h.size() * sizeof(float)), "h2d");
  crb::check(crb_dwa_control_many_batched(ctx, (int64_t)n, dx, dx + 5 * n, dx + 7 * n, dx + 9 * n, (int64_t)n_rows,
                                          (const int64_t*)d, (int32_t)n, (const int32_t*)(d + 2 * (n + 1)), &prm,
                                          nullptr, (int32_t*)dbest, dtraj, nullptr),
             "crb_dwa_control_many_batched");
  std::vector<float> hu(2 * n), tr(5 * (size_t)n_pts * n);
  std::vector<int32_t> best(n);
  crb::check(crb_memcpy_d2h(ctx, hu.data(), dx + 5 * n, hu.size() * sizeof(float)), "d2h");
  crb::check(crb_memcpy_d2h(ctx, best.data(), dbest, n * sizeof(int32_t)), "d2h");
  crb::check(crb_memcpy_d2h(ctx, tr.data(), dtraj, tr.size() * sizeof(float)), "d2h");
  for (size_t i = 0; i < n; ++i) {
    u[i][0] = hu[i];
    u[i][1] = hu[n + i];
    if (best[i] < 0) continue;
    out[i].resize((size_t)n_pts);
    for (int k = 0; k < n_pts; ++k)
      for (int j = 0; j < 5; ++j) out[i][(size_t)k][(size_t)j] = tr[(size_t)(5 * k + j) * n + i];
  }
  return out;
}

// dwa_control for a mixed fleet, each robot with its own Config and its own obstacles: robot i is dwa_control(x[i],
// u[i], config[i], goal[i], ob[i]) (u[i] set, its rollout of its own Config's length returned in element i, empty when
// no sample is admissible), all in one launch of crb_dwa_control_fleet_batched.  Bitwise-equal Configs share one
// record of the table.  A Config outside crb.h's limits throws before any device work.  Each ob[i] must have at most
// CRB_DWA_MAX_OBSTACLES rows.
template <class Config>
inline std::vector<std::vector<std::array<float, 5>>> dwa_control(
    const std::vector<std::array<float, 5>>& x, std::vector<std::array<float, 2>>& u,
    const std::vector<Config>& config, const std::vector<std::array<float, 2>>& goal,
    const std::vector<std::vector<std::array<float, 2>>>& ob) {
  const size_t n = x.size();
  if (u.size() != n || config.size() != n || goal.size() != n || ob.size() != n)
    throw std::runtime_error("dwa_control: x, u, config, goal and ob differ in length");
  std::vector<std::vector<std::array<float, 5>>> out(n);
  if (n == 0) return out;
  // the table: one record per bitwise-distinct Config, each checked here
  std::vector<crb_dwa_params> table;
  std::vector<int> n_pts;
  std::vector<int32_t> of(n);
  int max_pts = 0;
  for (size_t i = 0; i < n; ++i) {
    const crb_dwa_params prm = crb::dwa_params_of(config[i]);
    size_t c = 0;
    while (c < table.size() && std::memcmp(&table[c], &prm, sizeof(prm)) != 0) ++c;
    if (c == table.size()) {
      int k = 0;
      crb::check(crb_dwa_rollout_points(&prm, &k), "crb_dwa_rollout_points");
      table.push_back(prm);
      n_pts.push_back(k);
      max_pts = std::max(max_pts, k);
    }
    of[i] = (int32_t)c;
  }
  const size_t m = table.size();
  crb_ctx* ctx = crb::Session::get();
  // host: ob_off [n + 1] int64 | ob_of [n] int32 | config_of [n] int32 | x [5][n] | u [2][n] | goal [2][n] |
  //       table [m][12] | ob [n_rows][2]
  std::vector<int64_t> off(n + 1, 0);
  for (size_t i = 0; i < n; ++i) off[i + 1] = off[i] + (int64_t)ob[i].size();
  const size_t n_rows = (size_t)off[n];
  std::vector<float> h(2 * (n + 1) + 2 * n + 9 * n + 12 * m + 2 * n_rows);
  std::memcpy(h.data(), off.data(), off.size() * sizeof(int64_t));
  std::memcpy(h.data() + 2 * (n + 1) + n, of.data(), n * sizeof(int32_t));
  float* hx = h.data() + 4 * n + 2;
  std::memcpy(hx + 9 * n, table.data(), m * sizeof(crb_dwa_params));
  float* hob = hx + 9 * n + 12 * m;
  for (size_t i = 0; i < n; ++i) {
    const int32_t s = (int32_t)i;
    std::memcpy(h.data() + 2 * (n + 1) + i, &s, 4);
    for (int f = 0; f < 5; ++f) hx[f * n + i] = x[i][f];
    for (int f = 0; f < 2; ++f) hx[(5 + f) * n + i] = u[i][f];
    for (int f = 0; f < 2; ++f) hx[(7 + f) * n + i] = goal[i][f];
    for (size_t k = 0; k < ob[i].size(); ++k) {
      hob[2 * (off[i] + k)] = ob[i][k][0];
      hob[2 * (off[i] + k) + 1] = ob[i][k][1];
    }
  }
  // device: the host block | best [n] | traj [5 max_pts][n]; the arena comes from cudaMalloc, so ob_off is aligned
  float* d = crb::Session::scratch(h.size() + n + 5 * (size_t)max_pts * n);
  float *dx = d + 4 * n + 2, *dbest = d + h.size(), *dtraj = dbest + n;
  crb::check(crb_memcpy_h2d(ctx, d, h.data(), h.size() * sizeof(float)), "h2d");
  crb::check(crb_dwa_control_fleet_batched(ctx, (int64_t)n, dx, dx + 5 * n, dx + 7 * n,
                                           dx + 9 * n + 12 * m, (int64_t)n_rows, (const int64_t*)d, (int32_t)n,
                                           (const int32_t*)(d + 2 * (n + 1)), (const crb_dwa_params*)(dx + 9 * n),
                                           (int32_t)m, (const int32_t*)(d + 2 * (n + 1) + n), max_pts, nullptr,
                                           (int32_t*)dbest, dtraj, nullptr, nullptr),
             "crb_dwa_control_fleet_batched");
  std::vector<float> hu(2 * n), tr(5 * (size_t)max_pts * n);
  std::vector<int32_t> best(n);
  crb::check(crb_memcpy_d2h(ctx, hu.data(), dx + 5 * n, hu.size() * sizeof(float)), "d2h");
  crb::check(crb_memcpy_d2h(ctx, best.data(), dbest, n * sizeof(int32_t)), "d2h");
  crb::check(crb_memcpy_d2h(ctx, tr.data(), dtraj, tr.size() * sizeof(float)), "d2h");
  for (size_t i = 0; i < n; ++i) {
    u[i][0] = hu[i];
    u[i][1] = hu[n + i];
    if (best[i] < 0) continue;
    const int k_pts = n_pts[(size_t)of[i]];
    out[i].resize((size_t)k_pts);
    for (int k = 0; k < k_pts; ++k)
      for (int j = 0; j < 5; ++j) out[i][(size_t)k][(size_t)j] = tr[(size_t)(5 * k + j) * n + i];
  }
  return out;
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

// motion :43-50 for a fleet, each robot with its own dt (main()'s motion(x, u, config.dt) :194 with a Config per
// robot): robot i is motion(x[i], u[i], dt[i]), dt applied as given, all in one launch of crb_dwa_motion_fleet_batched.
inline std::vector<std::array<float, 5>> motion(std::vector<std::array<float, 5>> x,
                                                const std::vector<std::array<float, 2>>& u,
                                                const std::vector<float>& dt) {
  const size_t n = x.size();
  if (u.size() != n || dt.size() != n) throw std::runtime_error("motion: x, u and dt differ in length");
  if (n == 0) return x;
  crb_ctx* ctx = crb::Session::get();
  // x [5][n] | u [2][n] | dt [n]
  std::vector<float> h(8 * n);
  for (size_t i = 0; i < n; ++i) {
    for (int f = 0; f < 5; ++f) h[f * n + i] = x[i][f];
    for (int f = 0; f < 2; ++f) h[(5 + f) * n + i] = u[i][f];
    h[7 * n + i] = dt[i];
  }
  float* dx = crb::Session::scratch(h.size());
  crb::check(crb_memcpy_h2d(ctx, dx, h.data(), h.size() * sizeof(float)), "h2d");
  crb::check(crb_dwa_motion_fleet_batched(ctx, (int64_t)n, dx, dx + 5 * n, dx + 7 * n),
             "crb_dwa_motion_fleet_batched");
  crb::check(crb_memcpy_d2h(ctx, h.data(), dx, 5 * n * sizeof(float)), "d2h");
  for (size_t i = 0; i < n; ++i)
    for (int f = 0; f < 5; ++f) x[i][f] = h[f * n + i];
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

// src/state_lattice_planner.cpp:25-155 (its Table typedef, include/motion_model.h:56's StateList).  The samplers run
// one query through crb_slp_sample_states_batched; generate_path runs its whole list as one batch: one search launch
// and one optimizer launch, with crb_slp_default_params' settings (the file's L, DS, CONST_V, cost_th_, h_step_ and
// max_iter; no macro of those names is defined here).  A state whose search finds no row (the reference reads
// csv_file[-1]) or whose optimization stops with a status other than CONVERGED / MAX_ITER_REACHED throws.
using StateList = std::vector<TrajState>;
typedef std::vector<std::vector<float>> Table;

namespace detail {
// qp [nf] | target [3 S] | n_states, status  (n_q = 1)
inline StateList slp_sample(int kind, int nxy, int nh, int ns, int d, const float* qp, int nf) {
  crb_ctx* ctx = crb::Session::get();
  crb_slp_sampler s;
  s.kind = kind; s.nxy = nxy; s.nh = nh; s.ns = ns; s.d = d;
  const int S = crb_slp_states_per_query(&s);
  crb::check(S < 0 ? S : CRB_OK, "crb_slp_states_per_query");
  float* q = crb::Session::scratch(nf + 3 * (size_t)S + 2);
  float *t = q + nf, *cnt = t + 3 * (size_t)S;
  crb::check(crb_memcpy_h2d(ctx, q, qp, nf * sizeof(float)), "h2d");
  crb::check(crb_slp_sample_states_batched(ctx, 1, &s, q, t, (int32_t*)cnt, (int32_t*)(cnt + 1)),
             "crb_slp_sample_states_batched");
  int32_t ks[2];
  crb::check(crb_memcpy_d2h(ctx, ks, cnt, sizeof(ks)), "d2h");
  if (ks[1] != CRB_SLP_OK) throw std::runtime_error("state lattice sampler: an angle is outside the exact sin/cos range");
  std::vector<float> h(3 * (size_t)S);
  if (S) crb::check(crb_memcpy_d2h(ctx, h.data(), t, h.size() * sizeof(float)), "d2h");
  StateList states;
  for (int k = 0; k < ks[0]; ++k) states.push_back(TrajState(h[k], h[S + k], h[2 * (size_t)S + k]));
  return states;
}
inline std::vector<float> slp_flat_table(const Table& csv_file) {
  std::vector<float> t;
  t.reserve(6 * csv_file.size());
  for (size_t r = 0; r < csv_file.size(); ++r) {
    if (csv_file[r].size() < 6) throw std::runtime_error("lookup table: a row has fewer than 6 columns");
    t.insert(t.end(), csv_file[r].begin(), csv_file[r].begin() + 6);
  }
  if (t.empty() || csv_file.size() > 0x7fffffffu) throw std::runtime_error("lookup table: bad number of rows");
  return t;
}
}  // namespace detail

// calc_uniform_polar_states :47-56
inline StateList calc_uniform_polar_states(int nxy, int nh, int d, float a_min, float a_max, float p_min, float p_max) {
  const float qp[4] = {a_min, a_max, p_min, p_max};
  return detail::slp_sample(CRB_SLP_UNIFORM, nxy, nh, 0, d, qp, 4);
}
// calc_biased_polar_states :58-99
inline StateList calc_biased_polar_states(float goal_angle, int ns, int nxy, int nh, int d, float a_min, float a_max,
                                          float p_min, float p_max) {
  const float qp[5] = {goal_angle, a_min, a_max, p_min, p_max};
  return detail::slp_sample(CRB_SLP_BIASED, nxy, nh, ns, d, qp, 5);
}
// calc_lane_states :101-113
inline StateList calc_lane_states(float l_center, float l_heading, float l_width, float v_width, float d, int nxy) {
  const float qp[5] = {l_center, l_heading, l_width, v_width, d};
  return detail::slp_sample(CRB_SLP_LANE, nxy, 1, 0, 0, qp, 5);
}

// search_nearest_one_from_lookuptable :115-135: (|xy|, {0, km, kf}) of the nearest row
inline Parameter search_nearest_one_from_lookuptable(TrajState target, Table csv_file) {
  crb_ctx* ctx = crb::Session::get();
  const std::vector<float> tb = detail::slp_flat_table(csv_file);
  // table [6 rows] | target [3] | param [4] | row [1]
  float* dtb = crb::Session::scratch(tb.size() + 8);
  float *dt = dtb + tb.size(), *dp = dt + 3;
  const float t[3] = {target.x, target.y, target.yaw};
  crb::check(crb_memcpy_h2d(ctx, dtb, tb.data(), tb.size() * sizeof(float)), "h2d");
  crb::check(crb_memcpy_h2d(ctx, dt, t, sizeof(t)), "h2d");
  crb::check(crb_slp_search_nearest_batched(ctx, 1, dt, dtb, (int)csv_file.size(), nullptr, dp, (int32_t*)(dp + 4)),
             "crb_slp_search_nearest_batched");
  float p[5];
  crb::check(crb_memcpy_d2h(ctx, p, dp, sizeof(p)), "d2h");
  int32_t row;
  std::memcpy(&row, &p[4], sizeof(row));
  if (row < 0) throw std::runtime_error("search_nearest_one_from_lookuptable: no row is nearer than FLT_MAX");
  return Parameter(p[0], {{p[1], p[2], p[3]}});
}

// generate_path :137-155
inline std::vector<Traj> generate_path(StateList states, Table csv_file, float k0 = 0.0) {
  crb_ctx* ctx = crb::Session::get();
  const std::vector<float> tb = detail::slp_flat_table(csv_file);
  const size_t n = states.size();
  std::vector<Traj> out(n);
  if (n == 0) return out;
  crb_mptg_params prm;
  float v = 0.0f;
  crb_slp_default_params(&prm, &v);
  std::vector<float> h(8 * n, 0.0f);  // target [3][n] | k0 [n] | state [4][n]
  for (size_t i = 0; i < n; ++i) {
    h[i] = states[i].x;
    h[n + i] = states[i].y;
    h[2 * n + i] = states[i].yaw;
    h[3 * n + i] = k0;
    h[7 * n + i] = v;  // state (0, 0, 0, CONST_V)
  }
  int max_pts = 256;
  for (;;) {
    // target [3n] | k0 [n] | state [4n] | param [4n] | row, len, status [3n] | table | traj [3 max_pts n]
    float* d = crb::Session::scratch(15 * n + tb.size() + 3 * (size_t)max_pts * n);
    float *dk0 = d + 3 * n, *dst = dk0 + n, *dp = dst + 4 * n, *drow = dp + 4 * n, *dlen = drow + n,
          *dstat = dlen + n, *dtb = dstat + n, *dtraj = dtb + tb.size();
    crb::check(crb_memcpy_h2d(ctx, d, h.data(), 8 * n * sizeof(float)), "h2d");
    crb::check(crb_memcpy_h2d(ctx, dtb, tb.data(), tb.size() * sizeof(float)), "h2d");
    crb::check(crb_slp_search_nearest_batched(ctx, (int64_t)n, d, dtb, (int)csv_file.size(), dk0, dp,
                                              (int32_t*)drow),
               "crb_slp_search_nearest_batched");
    crb::check(crb_mptg_optimize_batched(ctx, (int64_t)n, dst, d, dp, &prm, max_pts, dtraj, (int32_t*)dlen, nullptr,
                                         (int32_t*)dstat, nullptr),
               "crb_mptg_optimize_batched");
    std::vector<int32_t> rls(3 * n);
    crb::check(crb_memcpy_d2h(ctx, rls.data(), drow, rls.size() * sizeof(int32_t)), "d2h");
    int longest = 0;
    for (size_t i = 0; i < n; ++i) {
      if (rls[i] < 0) throw std::runtime_error("generate_path: a state has no nearest lookup-table row");
      const int st = rls[2 * n + i];
      if (st != CRB_MPTG_CONVERGED && st != CRB_MPTG_MAX_ITER_REACHED)
        throw std::runtime_error("generate_path: optimizer_traj stopped with status " + std::to_string(st));
      if (rls[n + i] > longest) longest = rls[n + i];
    }
    if (longest > max_pts) {  // the same batch again with room for every whole trajectory
      max_pts = longest;
      continue;
    }
    std::vector<float> tr(3 * (size_t)max_pts * n);
    crb::check(crb_memcpy_d2h(ctx, tr.data(), dtraj, tr.size() * sizeof(float)), "d2h");
    for (size_t i = 0; i < n; ++i) {
      Traj& t = out[i];
      t.reserve((size_t)rls[n + i]);
      for (int k = 0; k < rls[n + i]; ++k)
        t.push_back(TrajState(tr[(3 * (size_t)k) * n + i], tr[(3 * (size_t)k + 1) * n + i],
                              tr[(3 * (size_t)k + 2) * n + i]));
    }
    return out;
  }
}
}  // namespace cpprobotics

// src/a_star.cpp:110-244 and src/dijkstra.cpp.  The reference's planners return nothing and draw; these return what
// its calc_final_path :31-45 computes, {rx, ry}: the goal first, then parent after parent down to the start, each
// cell * reso.  The batched overloads plan every (sx[i], sy[i], gx[i], gy[i]) on the one map of ox / oy in one
// launch and return one {rx, ry} per query.  A query the reference does not define (an unreachable goal, a start
// outside the box or a non-finite point: crb.h's CRB_GRID_* statuses) throws.
namespace cpprobotics {
namespace detail {
inline std::vector<std::vector<std::vector<float>>> grid_plan(int algo, const std::vector<float>& sx,
                                                              const std::vector<float>& sy,
                                                              const std::vector<float>& gx,
                                                              const std::vector<float>& gy,
                                                              const std::vector<float>& ox,
                                                              const std::vector<float>& oy, float reso, float rr) {
  crb_ctx* ctx = crb::Session::get();
  const size_t n = sx.size();
  if (sy.size() != n || gx.size() != n || gy.size() != n) throw std::runtime_error("grid planner: sx, sy, gx, gy differ in length");
  if (ox.size() != oy.size()) throw std::runtime_error("grid planner: ox and oy differ in length");
  crb_grid_box box;
  crb::check(crb_grid_box_of_obstacles((int64_t)ox.size(), ox.data(), oy.data(), reso, &box),
             "crb_grid_box_of_obstacles");
  std::vector<std::vector<std::vector<float>>> out(n);
  if (n == 0) return out;
  const size_t no = ox.size(), cells = (size_t)((int64_t)box.max_x - box.min_x) * (size_t)((int64_t)box.max_y - box.min_y);
  std::vector<float> h(2 * no + 4 * n);  // ox | oy | sg [4][n]
  std::copy(ox.begin(), ox.end(), h.begin());
  std::copy(oy.begin(), oy.end(), h.begin() + no);
  for (size_t i = 0; i < n; ++i) {
    h[2 * no + i] = sx[i];
    h[2 * no + n + i] = sy[i];
    h[2 * no + 2 * n + i] = gx[i];
    h[2 * no + 3 * n + i] = gy[i];
  }
  int max_pts = 256;
  for (;;) {
    // ox, oy, sg | len, status [2n] | map [cells bytes] | path [2 max_pts n]
    const size_t map_f = (cells + 3) / 4;
    float* d = crb::Session::scratch(h.size() + 2 * n + map_f + 2 * (size_t)max_pts * n);
    float *dsg = d + 2 * no, *dls = dsg + 4 * n, *dmap = dls + 2 * n, *dpath = dmap + map_f;
    crb::check(crb_memcpy_h2d(ctx, d, h.data(), h.size() * sizeof(float)), "h2d");
    crb::check(crb_grid_obstacle_map(ctx, (int64_t)no, d, d + no, reso, rr, &box, (uint8_t*)dmap),
               "crb_grid_obstacle_map");
    crb::check(crb_grid_plan_batched(ctx, algo, &box, (const uint8_t*)dmap, reso, (int64_t)n, dsg, max_pts, dpath,
                                     (int32_t*)dls, nullptr, nullptr, (int32_t*)(dls + n)),
               "crb_grid_plan_batched");
    std::vector<int32_t> ls(2 * n);
    crb::check(crb_memcpy_d2h(ctx, ls.data(), dls, ls.size() * sizeof(int32_t)), "d2h");
    int longest = 0;
    for (size_t i = 0; i < n; ++i) {
      if (ls[n + i] != CRB_GRID_FOUND)
        throw std::runtime_error("grid planner: no path (status " + std::to_string(ls[n + i]) + ")");
      if (ls[i] > longest) longest = ls[i];
    }
    if (longest > max_pts) {  // again with room for every whole path
      max_pts = longest;
      continue;
    }
    std::vector<float> p(2 * (size_t)max_pts * n);
    crb::check(crb_memcpy_d2h(ctx, p.data(), dpath, p.size() * sizeof(float)), "d2h");
    for (size_t i = 0; i < n; ++i) {
      std::vector<float> rx, ry;
      for (int k = 0; k < ls[i]; ++k) {
        rx.push_back(p[(2 * (size_t)k) * n + i]);
        ry.push_back(p[(2 * (size_t)k + 1) * n + i]);
      }
      out[i] = {rx, ry};
    }
    return out;
  }
}
}  // namespace detail

inline std::vector<std::vector<float>> a_star_planning(float sx, float sy, float gx, float gy, std::vector<float> ox_,
                                                       std::vector<float> oy_, float reso, float rr) {
  return detail::grid_plan(CRB_GRID_ASTAR, {sx}, {sy}, {gx}, {gy}, ox_, oy_, reso, rr)[0];
}
inline std::vector<std::vector<float>> dijkstra_star_planning(float sx, float sy, float gx, float gy,
                                                              std::vector<float> ox_, std::vector<float> oy_,
                                                              float reso, float rr) {
  return detail::grid_plan(CRB_GRID_DIJKSTRA, {sx}, {sy}, {gx}, {gy}, ox_, oy_, reso, rr)[0];
}
inline std::vector<std::vector<std::vector<float>>> a_star_planning(std::vector<float> sx, std::vector<float> sy,
                                                                    std::vector<float> gx, std::vector<float> gy,
                                                                    std::vector<float> ox_, std::vector<float> oy_,
                                                                    float reso, float rr) {
  return detail::grid_plan(CRB_GRID_ASTAR, sx, sy, gx, gy, ox_, oy_, reso, rr);
}
inline std::vector<std::vector<std::vector<float>>> dijkstra_star_planning(std::vector<float> sx, std::vector<float> sy,
                                                                           std::vector<float> gx, std::vector<float> gy,
                                                                           std::vector<float> ox_,
                                                                           std::vector<float> oy_, float reso,
                                                                           float rr) {
  return detail::grid_plan(CRB_GRID_DIJKSTRA, sx, sy, gx, gy, ox_, oy_, reso, rr);
}

// The same with a map per query: query i is exactly the reference call (sx[i], sy[i], gx[i], gy[i], ox_[i], oy_[i],
// reso[i], rr[i]).  Every query's map is built in one crb_grid_obstacle_map_many launch and every query planned in one
// crb_grid_plan_many_batched launch.  Throws as the overloads above do.
namespace detail {
inline std::vector<std::vector<std::vector<float>>> grid_plan_many(
    int algo, const std::vector<float>& sx, const std::vector<float>& sy, const std::vector<float>& gx,
    const std::vector<float>& gy, const std::vector<std::vector<float>>& ox, const std::vector<std::vector<float>>& oy,
    const std::vector<float>& reso, const std::vector<float>& rr) {
  crb_ctx* ctx = crb::Session::get();
  const size_t n = sx.size();
  if (sy.size() != n || gx.size() != n || gy.size() != n || ox.size() != n || oy.size() != n || reso.size() != n ||
      rr.size() != n)
    throw std::runtime_error("grid planner: the per-query arguments differ in length");
  std::vector<std::vector<std::vector<float>>> out(n);
  if (n == 0) return out;
  // host: map_off [n + 1] | ob_off [n + 1] (int64) | boxes [n][4] | ob_of [n] (int32) | reso | rr | sg [4][n] |
  // ob [n_rows][2]
  std::vector<int64_t> moff(n + 1, 0), ooff(n + 1, 0);
  std::vector<crb_grid_box> boxes(n);
  int64_t max_cells = 1;
  for (size_t i = 0; i < n; ++i) {
    if (ox[i].size() != oy[i].size()) throw std::runtime_error("grid planner: ox and oy differ in length");
    crb::check(crb_grid_box_of_obstacles((int64_t)ox[i].size(), ox[i].data(), oy[i].data(), reso[i], &boxes[i]),
               "crb_grid_box_of_obstacles");
    const int64_t cells = ((int64_t)boxes[i].max_x - boxes[i].min_x) * ((int64_t)boxes[i].max_y - boxes[i].min_y);
    if (cells > max_cells) max_cells = cells;
    moff[i + 1] = moff[i] + (cells > 0 ? cells : 0);
    ooff[i + 1] = ooff[i] + (int64_t)ox[i].size();
  }
  const size_t n_rows = (size_t)ooff[n], n_cells = (size_t)moff[n];
  const size_t o_box = 4 * (n + 1), o_of = o_box + 4 * n, o_reso = o_of + n, o_rr = o_reso + n, o_sg = o_rr + n,
               o_ob = o_sg + 4 * n;
  std::vector<float> h(o_ob + 2 * n_rows);
  std::memcpy(h.data(), moff.data(), moff.size() * sizeof(int64_t));
  std::memcpy(h.data() + 2 * (n + 1), ooff.data(), ooff.size() * sizeof(int64_t));
  std::memcpy(h.data() + o_box, boxes.data(), n * sizeof(crb_grid_box));
  for (size_t i = 0; i < n; ++i) {
    const int32_t s = (int32_t)i;
    std::memcpy(h.data() + o_of + i, &s, 4);
    h[o_reso + i] = reso[i];
    h[o_rr + i] = rr[i];
    h[o_sg + i] = sx[i];
    h[o_sg + n + i] = sy[i];
    h[o_sg + 2 * n + i] = gx[i];
    h[o_sg + 3 * n + i] = gy[i];
    for (size_t k = 0; k < ox[i].size(); ++k) {
      h[o_ob + 2 * ((size_t)ooff[i] + k)] = ox[i][k];
      h[o_ob + 2 * ((size_t)ooff[i] + k) + 1] = oy[i][k];
    }
  }
  int max_pts = 256;
  for (;;) {
    // device: the host block | len, status [2n] | maps [n_cells bytes] | path [2 max_pts n]
    const size_t map_f = (n_cells + 3) / 4;
    float* d = crb::Session::scratch(h.size() + 2 * n + map_f + 2 * (size_t)max_pts * n);
    float *dls = d + h.size(), *dmap = dls + 2 * n, *dpath = dmap + map_f;
    const int64_t* dmoff = (const int64_t*)d;
    const crb_grid_box* dbox = (const crb_grid_box*)(d + o_box);
    crb::check(crb_memcpy_h2d(ctx, d, h.data(), h.size() * sizeof(float)), "h2d");
    crb::check(crb_grid_obstacle_map_many(ctx, d + o_ob, (int64_t)n_rows, (const int64_t*)(d + 2 * (n + 1)),
                                          (int32_t)n, (const int32_t*)(d + o_of), d + o_rr, dbox, d + o_reso, dmoff,
                                          (int32_t)n, (int64_t)n_cells, max_cells, (uint8_t*)dmap, nullptr),
               "crb_grid_obstacle_map_many");
    crb::check(crb_grid_plan_many_batched(ctx, algo, dbox, d + o_reso, dmoff, (int32_t)n, (const uint8_t*)dmap,
                                          (int64_t)n_cells, max_cells, (int64_t)n, (const int32_t*)(d + o_of),
                                          d + o_sg, max_pts, dpath, (int32_t*)dls, nullptr, nullptr,
                                          (int32_t*)(dls + n)),
               "crb_grid_plan_many_batched");
    std::vector<int32_t> ls(2 * n);
    crb::check(crb_memcpy_d2h(ctx, ls.data(), dls, ls.size() * sizeof(int32_t)), "d2h");
    int longest = 0;
    for (size_t i = 0; i < n; ++i) {
      if (ls[n + i] != CRB_GRID_FOUND)
        throw std::runtime_error("grid planner: no path (status " + std::to_string(ls[n + i]) + ")");
      if (ls[i] > longest) longest = ls[i];
    }
    if (longest > max_pts) {  // again with room for every whole path
      max_pts = longest;
      continue;
    }
    std::vector<float> p(2 * (size_t)max_pts * n);
    crb::check(crb_memcpy_d2h(ctx, p.data(), dpath, p.size() * sizeof(float)), "d2h");
    for (size_t i = 0; i < n; ++i) {
      std::vector<float> rx, ry;
      for (int k = 0; k < ls[i]; ++k) {
        rx.push_back(p[(2 * (size_t)k) * n + i]);
        ry.push_back(p[(2 * (size_t)k + 1) * n + i]);
      }
      out[i] = {rx, ry};
    }
    return out;
  }
}
}  // namespace detail

inline std::vector<std::vector<std::vector<float>>> a_star_planning(
    std::vector<float> sx, std::vector<float> sy, std::vector<float> gx, std::vector<float> gy,
    std::vector<std::vector<float>> ox_, std::vector<std::vector<float>> oy_, std::vector<float> reso,
    std::vector<float> rr) {
  return detail::grid_plan_many(CRB_GRID_ASTAR, sx, sy, gx, gy, ox_, oy_, reso, rr);
}
inline std::vector<std::vector<std::vector<float>>> dijkstra_star_planning(
    std::vector<float> sx, std::vector<float> sy, std::vector<float> gx, std::vector<float> gy,
    std::vector<std::vector<float>> ox_, std::vector<std::vector<float>> oy_, std::vector<float> reso,
    std::vector<float> rr) {
  return detail::grid_plan_many(CRB_GRID_DIJKSTRA, sx, sy, gx, gy, ox_, oy_, reso, rr);
}
}  // namespace cpprobotics

// include/rrt.h:21-159.  Node has the reference's members and constructor.  RRT has its constructor (path_resolution is
// kept and unused, as there) and planning() returns what the reference's does: end, then the last node and its parents
// down to, not including, the start, then start, each node's parent the next element (end's and start's stay NULL).
// goal_gen is seeded from std::random_device as in the reference; seed(s) makes the next planning() call the
// reference's after goal_gen.seed(s).  The reference loops until it finds a path and ignores max_iter; here max_iter
// is raised to CRB_RRT_MAX_ITER and a query that is not FOUND within it (crb.h's CRB_RRT_* statuses) throws.  The
// batched overload plans every (starts[i], ends[i]) with goal_gen.seed(seeds[i]) on this RRT's obstacles in one
// launch; the overload with ob_lists plans query i among ob_lists[i] instead (as an RRT constructed with that list),
// all in one launch of crb_rrt_plan_many_batched.  The RRT object owns the nodes it returns (the reference leaks them).
namespace cpprobotics {
class Node {
 public:
  float x;
  float y;
  std::vector<float> path_x;
  std::vector<float> path_y;
  Node* parent;
  float cost;
  Node(float x_, float y_) : x(x_), y(y_), parent(NULL), cost(0) {}
};

class RRT {
 public:
  RRT(Node* start_, Node* end_, std::vector<std::vector<float> > ob_list_, std::vector<float> rand_area_,
      float expand_dis_ = 1.0, float path_resolution_ = 1.0, int goal_sample_rate_ = 5, int max_iter_ = 500)
      : start(start_), end(end_), expand_dis(expand_dis_), path_resolution(path_resolution_),
        goal_sample_rate(goal_sample_rate_), max_iter(max_iter_), ob_list(ob_list_), rand_area(rand_area_),
        next_seed(std::random_device()()) {
    if (rand_area.size() != 2) throw std::runtime_error("RRT: rand_area needs {min, max}");
  }
  // the next planning() is the reference's after goal_gen.seed(s)
  void seed(uint32_t s) { next_seed = s; }

  std::vector<Node*> planning() {
    std::vector<std::vector<Node*> > r = planning({start}, {end}, {next_seed});
    next_seed = std::random_device()();
    return r[0];
  }

  std::vector<std::vector<Node*> > planning(const std::vector<Node*>& starts, const std::vector<Node*>& ends,
                                            const std::vector<uint32_t>& seeds) {
    return plan(starts, ends, seeds, nullptr);
  }

  std::vector<std::vector<Node*> > planning(const std::vector<Node*>& starts, const std::vector<Node*>& ends,
                                            const std::vector<uint32_t>& seeds,
                                            const std::vector<std::vector<std::vector<float> > >& ob_lists) {
    if (ob_lists.size() != starts.size()) throw std::runtime_error("RRT: starts and ob_lists differ in length");
    return plan(starts, ends, seeds, &ob_lists);
  }

 protected:
  // lists NULL: every query on ob_list (crb_rrt_plan_batched); else query i on (*lists)[i] (crb_rrt_plan_many_batched)
  std::vector<std::vector<Node*> > plan(const std::vector<Node*>& starts, const std::vector<Node*>& ends,
                                        const std::vector<uint32_t>& seeds,
                                        const std::vector<std::vector<std::vector<float> > >* lists) {
    const size_t n = starts.size();
    if (ends.size() != n || seeds.size() != n) throw std::runtime_error("RRT: starts, ends, seeds differ in length");
    std::vector<std::vector<Node*> > out(n);
    if (n == 0) return out;
    crb_ctx* ctx = crb::Session::get();
    crb_rrt_params prm;
    prm.rand_min = rand_area[0];
    prm.rand_max = rand_area[1];
    prm.expand_dis = expand_dis;
    prm.goal_sample_rate = goal_sample_rate;
    prm.max_iter = CRB_RRT_MAX_ITER;
    // the rows: ob_list, or every query's list back to back with ob_off [n + 1] (int64) and ob_of [n] = i after them
    std::vector<const std::vector<std::vector<float> >*> src(1, &ob_list);
    if (lists) {
      src.clear();
      for (size_t i = 0; i < n; ++i) src.push_back(&(*lists)[i]);
    }
    std::vector<int64_t> off(1, 0);
    for (size_t i = 0; i < src.size(); ++i) off.push_back(off.back() + (int64_t)src[i]->size());
    const size_t no = (size_t)off.back();
    const size_t store = lists ? 2 * (n + 1) + n : 0;
    std::vector<float> h(3 * no + 5 * n + store);  // ob [no][3] | se [4][n] | seed [n] | ob_off, ob_of (per query)
    for (size_t i = 0; i < src.size(); ++i)
      for (size_t j = 0; j < src[i]->size(); ++j) {
        const std::vector<float>& o = (*src[i])[j];
        if (o.size() < 3) throw std::runtime_error("RRT: an obstacle needs {x, y, r}");
        for (int c = 0; c < 3; ++c) h[3 * (off[i] + j) + c] = o[c];
      }
    if (lists) {
      float* tail = h.data() + 3 * no + 5 * n;
      std::memcpy(tail, off.data(), off.size() * sizeof(int64_t));
      for (size_t i = 0; i < n; ++i) {
        const int32_t s = (int32_t)i;
        std::memcpy(tail + 2 * (n + 1) + i, &s, 4);
      }
    }
    for (size_t i = 0; i < n; ++i) {
      h[3 * no + i] = starts[i]->x;
      h[3 * no + n + i] = starts[i]->y;
      h[3 * no + 2 * n + i] = ends[i]->x;
      h[3 * no + 3 * n + i] = ends[i]->y;
      std::memcpy(&h[3 * no + 4 * n + i], &seeds[i], 4);
    }
    int max_pts = 256;
    for (;;) {
      // ob [no][3] | ob_off, ob_of | se, seed | len, status [2n] | path [2 max_pts n]; ob_off starts at an even
      // float index of the (cudaMalloc-aligned) scratch arena, so it is 8-byte aligned
      const size_t ob_floats = (3 * no + 1) / 2 * 2;
      float* d = crb::Session::scratch(ob_floats + store + 5 * n + 2 * n + 2 * (size_t)max_pts * n);
      float *dstore = d + ob_floats, *dse = dstore + store, *dls = dse + 5 * n, *dpath = dls + 2 * n;
      crb::check(crb_memcpy_h2d(ctx, d, h.data(), 3 * no * sizeof(float)), "h2d");
      crb::check(crb_memcpy_h2d(ctx, dse, h.data() + 3 * no, 5 * n * sizeof(float)), "h2d");
      if (lists) {
        crb::check(crb_memcpy_h2d(ctx, dstore, h.data() + 3 * no + 5 * n, store * sizeof(float)), "h2d");
        crb::check(crb_rrt_plan_many_batched(ctx, &prm, d, (int64_t)no, (const int64_t*)dstore, (int32_t)n,
                                             (const int32_t*)(dstore + 2 * (n + 1)), (int64_t)n, dse,
                                             (const uint32_t*)(dse + 4 * n), max_pts, dpath, (int32_t*)dls, 0,
                                             nullptr, nullptr, nullptr, nullptr, (int32_t*)(dls + n)),
                   "crb_rrt_plan_many_batched");
      } else {
        crb::check(crb_rrt_plan_batched(ctx, &prm, d, (int32_t)no, (int64_t)n, dse, (const uint32_t*)(dse + 4 * n),
                                        max_pts, dpath, (int32_t*)dls, 0, nullptr, nullptr, nullptr, nullptr,
                                        (int32_t*)(dls + n)),
                   "crb_rrt_plan_batched");
      }
      std::vector<int32_t> ls(2 * n);
      crb::check(crb_memcpy_d2h(ctx, ls.data(), dls, ls.size() * sizeof(int32_t)), "d2h");
      int longest = 0;
      for (size_t i = 0; i < n; ++i) {
        if (ls[n + i] != CRB_RRT_FOUND)
          throw std::runtime_error("RRT::planning: no path (status " + std::to_string(ls[n + i]) + ")");
        if (ls[i] > longest) longest = ls[i];
      }
      if (longest > max_pts) {  // again with room for every whole path
        max_pts = longest;
        continue;
      }
      std::vector<float> p(2 * (size_t)max_pts * n);
      crb::check(crb_memcpy_d2h(ctx, p.data(), dpath, p.size() * sizeof(float)), "d2h");
      for (size_t i = 0; i < n; ++i) {
        std::vector<Node*>& path = out[i];
        path.push_back(ends[i]);
        for (int k = 1; k + 1 < ls[i]; ++k) {
          owned.emplace_back(new Node(p[(2 * (size_t)k) * n + i], p[(2 * (size_t)k + 1) * n + i]));
          path.push_back(owned.back().get());
        }
        path.push_back(starts[i]);
        for (size_t k = 1; k + 1 < path.size(); ++k) path[k]->parent = path[k + 1];
      }
      return out;
    }
  }

  Node* start;
  Node* end;
  const float expand_dis;
  const float path_resolution;
  const int goal_sample_rate;
  const int max_iter;
  const std::vector<std::vector<float> > ob_list;
  std::vector<float> rand_area;
  uint32_t next_seed;
  std::vector<std::unique_ptr<Node> > owned;
};
}  // namespace cpprobotics

// ---------------------------------------------------------------------------------------------------
// LQR path tracking: src/lqr_steer_control.cpp and src/lqr_speed_steer_control.cpp.  Each program's functions live
// in a namespace named after it, because both programs and the MPC program (above) define update() with one
// signature; a main() written against one program says `using namespace cpprobotics::lqr_steer_control;` and calls
// lqr_steering_control(...) and lqr_steer_control::update(...).  calc_nearest_index runs inside lqr_steering_control.
// The single-vehicle calls copy the course to the device on every call, as the reference copies its vectors by value;
// the batched overloads take a fleet at once, on one course or with a course per vehicle.
// ---------------------------------------------------------------------------------------------------
namespace cpprobotics {
namespace detail {
// one control call for n vehicles on host arrays (AoS State), through the session's device arena
inline void lqr_control(int nx, const std::vector<State>& st, const Vec_f& cx, const Vec_f& cy, const Vec_f& cyaw,
                        const Vec_f& ck, const Vec_f* sp, int32_t* ind, float* pe, float* pth_e, float* u) {
  const int64_t n = (int64_t)st.size();
  const size_t nc = cx.size();
  if (nc == 0 || cy.size() != nc || cyaw.size() != nc || ck.size() != nc || (sp && sp->size() != nc))
    throw std::runtime_error("lqr_steering_control: the course vectors must be non-empty and of one length");
  if (n == 0) return;
  const int nu = nx == 4 ? 1 : 2;
  const size_t nn = (size_t)n;
  // layout: course (4 or 5 x nc) | state 4n | ind n | pe n | pth_e n | u nu*n
  const size_t need = (sp ? 5 : 4) * nc + (4 + 3 + nu) * nn;
  crb_ctx* ctx = crb::Session::get();
  float* base = crb::Session::scratch(need);
  float* dcx = base;
  float* dcy = dcx + nc;
  float* dcyaw = dcy + nc;
  float* dck = dcyaw + nc;
  float* dsp = sp ? dck + nc : nullptr;
  float* dst = dck + nc + (sp ? nc : 0);
  int32_t* dind = (int32_t*)(dst + 4 * nn);
  float* dpe = (float*)(dind + nn);
  float* dpth = dpe + nn;
  float* du = dpth + nn;
  std::vector<float> soa(4 * nn);
  for (size_t i = 0; i < nn; ++i) {
    soa[i] = st[i].x; soa[nn + i] = st[i].y; soa[2 * nn + i] = st[i].yaw; soa[3 * nn + i] = st[i].v;
  }
  crb::check(crb_memcpy_h2d(ctx, dcx, cx.data(), nc * 4), "crb_memcpy_h2d");
  crb::check(crb_memcpy_h2d(ctx, dcy, cy.data(), nc * 4), "crb_memcpy_h2d");
  crb::check(crb_memcpy_h2d(ctx, dcyaw, cyaw.data(), nc * 4), "crb_memcpy_h2d");
  crb::check(crb_memcpy_h2d(ctx, dck, ck.data(), nc * 4), "crb_memcpy_h2d");
  if (sp) crb::check(crb_memcpy_h2d(ctx, dsp, sp->data(), nc * 4), "crb_memcpy_h2d");
  crb::check(crb_memcpy_h2d(ctx, dst, soa.data(), soa.size() * 4), "crb_memcpy_h2d");
  crb::check(crb_memcpy_h2d(ctx, dind, ind, nn * 4), "crb_memcpy_h2d");
  crb::check(crb_memcpy_h2d(ctx, dpe, pe, nn * 4), "crb_memcpy_h2d");
  crb::check(crb_memcpy_h2d(ctx, dpth, pth_e, nn * 4), "crb_memcpy_h2d");
  crb_lqr_track_params prm;
  crb_lqr_track_default_params(&prm, nx);
  crb::check(crb_lqr_steering_control_batched(ctx, n, nx, dst, dcx, dcy, dcyaw, dck, dsp, (int32_t)nc, &prm, dind, dpe,
                                              dpth, du, nullptr, nullptr, nullptr),
             "crb_lqr_steering_control_batched");
  crb::check(crb_memcpy_d2h(ctx, ind, dind, nn * 4), "crb_memcpy_d2h");
  crb::check(crb_memcpy_d2h(ctx, pe, dpe, nn * 4), "crb_memcpy_d2h");
  crb::check(crb_memcpy_d2h(ctx, pth_e, dpth, nn * 4), "crb_memcpy_d2h");
  crb::check(crb_memcpy_d2h(ctx, u, du, nu * nn * 4), "crb_memcpy_d2h");
}
// one control call for n vehicles, vehicle i on its own course (cx[i], cy[i], ...), through the session's device arena:
// the courses packed back to back with one int64 offset per course, course_of[i] = i
inline void lqr_control_many(int nx, const std::vector<State>& st, const std::vector<Vec_f>& cx,
                             const std::vector<Vec_f>& cy, const std::vector<Vec_f>& cyaw, const std::vector<Vec_f>& ck,
                             const std::vector<Vec_f>* sp, int32_t* ind, float* pe, float* pth_e, float* u) {
  const size_t nn = st.size();
  if (cx.size() != nn || cy.size() != nn || cyaw.size() != nn || ck.size() != nn || (sp && sp->size() != nn))
    throw std::runtime_error("lqr_steering_control: one course per state");
  std::vector<int64_t> off(nn + 1, 0);
  for (size_t i = 0; i < nn; ++i) {
    const size_t nc = cx[i].size();
    if (nc == 0 || cy[i].size() != nc || cyaw[i].size() != nc || ck[i].size() != nc || (sp && (*sp)[i].size() != nc))
      throw std::runtime_error("lqr_steering_control: each course's vectors must be non-empty and of one length");
    off[i + 1] = off[i] + (int64_t)nc;
  }
  if (nn == 0) return;
  const int nu = nx == 4 ? 1 : 2;
  const size_t np = (size_t)off[nn];
  const int nf = sp ? 5 : 4;
  // layout: course_off (n+1) int64 | course fields (nf x np) | state 4n | ind n | pe n | pth_e n | u nu*n | course_of n
  const size_t need = 2 * (nn + 1) + nf * np + (4 + 3 + nu + 1) * nn;
  crb_ctx* ctx = crb::Session::get();
  float* arena = crb::Session::scratch(need);
  int64_t* doff = (int64_t*)arena;
  float* base = arena + 2 * (nn + 1);
  const std::vector<Vec_f>* fields[5] = {&cx, &cy, &cyaw, &ck, sp};
  std::vector<float> packed(np);
  for (int f = 0; f < nf; ++f) {
    for (size_t i = 0; i < nn; ++i) std::copy((*fields[f])[i].begin(), (*fields[f])[i].end(), packed.begin() + off[i]);
    crb::check(crb_memcpy_h2d(ctx, base + f * np, packed.data(), np * 4), "crb_memcpy_h2d");
  }
  float* dst = base + nf * np;
  int32_t* dind = (int32_t*)(dst + 4 * nn);
  float* dpe = (float*)(dind + nn);
  float* dpth = dpe + nn;
  float* du = dpth + nn;
  int32_t* dof = (int32_t*)(du + nu * nn);
  std::vector<float> soa(4 * nn);
  std::vector<int32_t> course_of(nn);
  for (size_t i = 0; i < nn; ++i) {
    soa[i] = st[i].x; soa[nn + i] = st[i].y; soa[2 * nn + i] = st[i].yaw; soa[3 * nn + i] = st[i].v;
    course_of[i] = (int32_t)i;
  }
  crb::check(crb_memcpy_h2d(ctx, dst, soa.data(), soa.size() * 4), "crb_memcpy_h2d");
  crb::check(crb_memcpy_h2d(ctx, dind, ind, nn * 4), "crb_memcpy_h2d");
  crb::check(crb_memcpy_h2d(ctx, dpe, pe, nn * 4), "crb_memcpy_h2d");
  crb::check(crb_memcpy_h2d(ctx, dpth, pth_e, nn * 4), "crb_memcpy_h2d");
  crb::check(crb_memcpy_h2d(ctx, dof, course_of.data(), nn * 4), "crb_memcpy_h2d");
  crb::check(crb_memcpy_h2d(ctx, doff, off.data(), (nn + 1) * 8), "crb_memcpy_h2d");
  crb_lqr_track_params prm;
  crb_lqr_track_default_params(&prm, nx);
  crb::check(crb_lqr_steering_control_many_batched(ctx, (int64_t)nn, nx, dst, base, base + np, base + 2 * np,
                                                   base + 3 * np, sp ? base + 4 * np : nullptr, doff, (int32_t)nn,
                                                   (int64_t)np, dof, &prm, dind, dpe, dpth, du, nullptr, nullptr,
                                                   nullptr),
             "crb_lqr_steering_control_many_batched");
  crb::check(crb_memcpy_d2h(ctx, ind, dind, nn * 4), "crb_memcpy_d2h");
  crb::check(crb_memcpy_d2h(ctx, pe, dpe, nn * 4), "crb_memcpy_d2h");
  crb::check(crb_memcpy_d2h(ctx, pth_e, dpth, nn * 4), "crb_memcpy_d2h");
  crb::check(crb_memcpy_d2h(ctx, u, du, nu * nn * 4), "crb_memcpy_d2h");
}
// update() of the LQR programs for n vehicles, in place
inline void lqr_update(std::vector<State>& st, const Vec_f& a, const Vec_f& delta) {
  const size_t nn = st.size();
  if (a.size() != nn || delta.size() != nn) throw std::runtime_error("update: a and delta need one value per state");
  if (nn == 0) return;
  crb_ctx* ctx = crb::Session::get();
  float* dst = crb::Session::scratch(6 * nn);
  float* da = dst + 4 * nn;
  float* dd = da + nn;
  std::vector<float> soa(4 * nn);
  for (size_t i = 0; i < nn; ++i) {
    soa[i] = st[i].x; soa[nn + i] = st[i].y; soa[2 * nn + i] = st[i].yaw; soa[3 * nn + i] = st[i].v;
  }
  crb::check(crb_memcpy_h2d(ctx, dst, soa.data(), soa.size() * 4), "crb_memcpy_h2d");
  crb::check(crb_memcpy_h2d(ctx, da, a.data(), nn * 4), "crb_memcpy_h2d");
  crb::check(crb_memcpy_h2d(ctx, dd, delta.data(), nn * 4), "crb_memcpy_h2d");
  crb_lqr_track_params prm;
  crb_lqr_track_default_params(&prm, 4);  // update is the same text in both programs
  crb::check(crb_lqr_update_batched(ctx, (int64_t)nn, dst, da, dd, &prm), "crb_lqr_update_batched");
  crb::check(crb_memcpy_d2h(ctx, soa.data(), dst, soa.size() * 4), "crb_memcpy_d2h");
  for (size_t i = 0; i < nn; ++i) {
    st[i].x = soa[i]; st[i].y = soa[nn + i]; st[i].yaw = soa[2 * nn + i]; st[i].v = soa[3 * nn + i];
  }
}
}  // namespace detail

namespace lqr_steer_control {
// src/lqr_steer_control.cpp:98-133: ind, pe, pth_e carry over between calls; returns delta
inline float lqr_steering_control(State state, Vec_f cx, Vec_f cy, Vec_f cyaw, Vec_f ck, int& ind, float& pe,
                                  float& pth_e) {
  int32_t i = ind;
  float delta = 0.0f;
  detail::lqr_control(4, std::vector<State>(1, state), cx, cy, cyaw, ck, nullptr, &i, &pe, &pth_e, &delta);
  ind = i;
  return delta;
}
// a fleet on one course: ind, pe, pth_e one per state (in/out); returns delta per state
inline Vec_f lqr_steering_control(const std::vector<State>& states, const Vec_f& cx, const Vec_f& cy,
                                  const Vec_f& cyaw, const Vec_f& ck, std::vector<int>& ind, Vec_f& pe, Vec_f& pth_e) {
  const size_t n = states.size();
  if (ind.size() != n || pe.size() != n || pth_e.size() != n)
    throw std::runtime_error("lqr_steering_control: ind, pe and pth_e need one value per state");
  std::vector<int32_t> i32(ind.begin(), ind.end());
  Vec_f delta(n);
  detail::lqr_control(4, states, cx, cy, cyaw, ck, nullptr, i32.data(), pe.data(), pth_e.data(), delta.data());
  for (size_t i = 0; i < n; ++i) ind[i] = i32[i];
  return delta;
}
// a fleet with a course per vehicle: state i follows (cx[i], cy[i], cyaw[i], ck[i]); ind (course-local), pe, pth_e
// one per state (in/out); returns delta per state
inline Vec_f lqr_steering_control(const std::vector<State>& states, const std::vector<Vec_f>& cx,
                                  const std::vector<Vec_f>& cy, const std::vector<Vec_f>& cyaw,
                                  const std::vector<Vec_f>& ck, std::vector<int>& ind, Vec_f& pe, Vec_f& pth_e) {
  const size_t n = states.size();
  if (ind.size() != n || pe.size() != n || pth_e.size() != n)
    throw std::runtime_error("lqr_steering_control: ind, pe and pth_e need one value per state");
  std::vector<int32_t> i32(ind.begin(), ind.end());
  Vec_f delta(n);
  detail::lqr_control_many(4, states, cx, cy, cyaw, ck, nullptr, i32.data(), pe.data(), pth_e.data(), delta.data());
  for (size_t i = 0; i < n; ++i) ind[i] = i32[i];
  return delta;
}
// :136-146
inline void update(State& state, float a, float delta) {
  std::vector<State> s(1, state);
  detail::lqr_update(s, Vec_f(1, a), Vec_f(1, delta));
  state = s[0];
}
inline void update(std::vector<State>& states, const Vec_f& a, const Vec_f& delta) { detail::lqr_update(states, a, delta); }
}  // namespace lqr_steer_control

namespace lqr_speed_steer_control {
// src/lqr_speed_steer_control.cpp:108-151: returns {ai, delta}; pe, pth_e carry over between calls
inline Vec_f lqr_steering_control(State state, Vec_f cx, Vec_f cy, Vec_f cyaw, Vec_f ck, Vec_f sp, float& pe,
                                  float& pth_e) {
  int32_t ind = 0;
  float u[2];
  detail::lqr_control(5, std::vector<State>(1, state), cx, cy, cyaw, ck, &sp, &ind, &pe, &pth_e, u);
  return Vec_f{u[0], u[1]};
}
// a fleet on one course: pe, pth_e one per state (in/out); returns {ai, delta} per state
inline std::vector<Vec_f> lqr_steering_control(const std::vector<State>& states, const Vec_f& cx, const Vec_f& cy,
                                               const Vec_f& cyaw, const Vec_f& ck, const Vec_f& sp, Vec_f& pe,
                                               Vec_f& pth_e) {
  const size_t n = states.size();
  if (pe.size() != n || pth_e.size() != n)
    throw std::runtime_error("lqr_steering_control: pe and pth_e need one value per state");
  std::vector<int32_t> ind(n, 0);
  Vec_f u(2 * n);
  detail::lqr_control(5, states, cx, cy, cyaw, ck, &sp, ind.data(), pe.data(), pth_e.data(), u.data());
  std::vector<Vec_f> out(n);
  for (size_t i = 0; i < n; ++i) out[i] = Vec_f{u[i], u[n + i]};
  return out;
}
// a fleet with a course per vehicle: state i follows (cx[i], cy[i], cyaw[i], ck[i], sp[i]); pe, pth_e one per state
// (in/out); returns {ai, delta} per state
inline std::vector<Vec_f> lqr_steering_control(const std::vector<State>& states, const std::vector<Vec_f>& cx,
                                               const std::vector<Vec_f>& cy, const std::vector<Vec_f>& cyaw,
                                               const std::vector<Vec_f>& ck, const std::vector<Vec_f>& sp, Vec_f& pe,
                                               Vec_f& pth_e) {
  const size_t n = states.size();
  if (pe.size() != n || pth_e.size() != n)
    throw std::runtime_error("lqr_steering_control: pe and pth_e need one value per state");
  std::vector<int32_t> ind(n, 0);
  Vec_f u(2 * n);
  detail::lqr_control_many(5, states, cx, cy, cyaw, ck, &sp, ind.data(), pe.data(), pth_e.data(), u.data());
  std::vector<Vec_f> out(n);
  for (size_t i = 0; i < n; ++i) out[i] = Vec_f{u[i], u[n + i]};
  return out;
}
// :154-164
inline void update(State& state, float a, float delta) { lqr_steer_control::update(state, a, delta); }
inline void update(std::vector<State>& states, const Vec_f& a, const Vec_f& delta) { detail::lqr_update(states, a, delta); }
}  // namespace lqr_speed_steer_control
}  // namespace cpprobotics

#endif  // CRB_REFERENCE_API_HPP_
