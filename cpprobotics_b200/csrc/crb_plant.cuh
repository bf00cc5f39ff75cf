// crb_plant.cuh — the kinematic bicycle step update(State&, a, delta) as the reference writes it in
// src/model_predictive_control.cpp:69-81 and, with the same text minus the speed clamp, in src/lqr_steer_control.cpp
// :136-146 and src/lqr_speed_steer_control.cpp:154-164.  Shared by crb_mpc_plant_update_kernel (crb_mpc.cu) and
// crb_lqr_update_kernel (crb_lqr_track.cu).
#pragma once
#include "crb_common.cuh"

// MAX_STEER, DT, WB (L), MAX_SPEED, MIN_SPEED are double macros in the reference, so the float operands promote to
// double and the results narrow on assignment; cos / sin / tan are the float overloads.  A program without a speed
// clamp passes +-inf as the speed bounds, which makes the clamp a no-op (NaN included).
struct PlantC {
  double max_steer, dt, wb, max_speed, min_speed;
};

__device__ __forceinline__ void crb_plant_step(float& x, float& y, float& yaw, float& v, float a, float delta,
                                               const PlantC& k) {
  const double MAX_STEER = k.max_steer, DT = k.dt, WB = k.wb;
  const double MAX_SPEED = k.max_speed, MIN_SPEED = k.min_speed;
  if ((double)delta >= MAX_STEER) delta = (float)MAX_STEER;
  if ((double)delta <= -MAX_STEER) delta = (float)(-MAX_STEER);
  float sy, cy;
  crb_sincosf_libm(yaw, sy, cy);   // std::cos / std::sin of a float: the host libm's bits (crb_common.cuh)
  const float nx = (float)((double)x + (double)(v * cy) * DT);
  const float ny = (float)((double)y + (double)(v * sy) * DT);
  // std::tan of a float: glibc's bits.  |delta| <= |max_steer| < 120 (checked on the host), inside crb_tanf_libm's
  // proven range; a NaN delta stays NaN
  const float nyaw = (float)((double)yaw + (double)v / WB * (double)crb_tanf_libm(delta) * DT);
  float nv = (float)((double)v + (double)a * DT);
  if ((double)nv > MAX_SPEED) nv = (float)MAX_SPEED;
  if ((double)nv < MIN_SPEED) nv = (float)MIN_SPEED;
  x = nx; y = ny; yaw = nyaw; v = nv;
}
