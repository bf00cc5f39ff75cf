// crb_dwa_common.cuh — the dynamic window approach's per-robot body and parameter check, shared by the single-Config
// kernels (crb_dwa.cu) and the Config-table kernels (crb_dwa_fleet.cu).  Both run this one dwa_robot, which is what
// makes a robot of the table entry bitwise the single-Config entry run with its Config, and both decide a Config with
// this one dwa_params_fault, on the host for a crb_dwa_params argument and on the device for a table record.
#pragma once
#include <float.h>
#include <math.h>

#include "crb_common.cuh"

#define DWA_BLOCK 256
#define DWA_WARPS (DWA_BLOCK / 32)

// motion() :43-50: yaw first, then the position with the NEW yaw, two separate float multiplies per axis.
__device__ __forceinline__ void crb_dwa_motion(float (&s)[5], float v, float w, float dt) {
  s[2] = s[2] + w * dt;
  float sn, cs;
  crb_sincosf_libm(s[2], sn, cs);
  s[0] = s[0] + v * cs * dt;
  s[1] = s[1] + v * sn * dt;
  s[3] = v;
  s[4] = w;
}

// glibc's acosf (the reference's std::acos(float), :109).  glibc 2.39 computes it with fdlibm's binary32
// algorithm (e_acosf.c, Sun Microsystems, freely redistributable): a rational approximation in z = x^2 or
// (1 - |x|) / 2 with three branches and, for x > 0.5, sqrtf(z) split at bit 12 so that 2 (df + w) keeps the
// extra precision.  Restated operation for operation; CUDA's own acosf rounds differently on ~5e6 inputs in
// [-1, 1].  |x| > 1 and NaN give NaN (its bits are not specified: a NaN cost never wins the selection).
__device__ __noinline__ inline float crb_dwa_acosf(float x) {  // inline: one host stub across the TUs
  const float pi = 3.1415925026e+00f, pio2_hi = 1.5707962513e+00f, pio2_lo = 7.5497894159e-08f;
  const float pS0 = 1.6666667163e-01f, pS1 = -3.2556581497e-01f, pS2 = 2.0121252537e-01f,
              pS3 = -4.0055535734e-02f, pS4 = 7.9153501429e-04f, pS5 = 3.4793309169e-05f;
  const float qS1 = -2.4033949375e+00f, qS2 = 2.0209457874e+00f, qS3 = -6.8828397989e-01f,
              qS4 = 7.7038154006e-02f;
  const int hx = __float_as_int(x);
  const int ix = hx & 0x7fffffff;
  if (ix == 0x3f800000) return hx > 0 ? 0.0f : pi + 2.0f * pio2_lo;  // |x| == 1
  if (ix > 0x3f800000) return (x - x) / (x - x);                      // |x| > 1, inf, NaN
  if (ix < 0x3f000000) {                                               // |x| < 0.5
    if (ix <= 0x23000000) return pio2_hi + pio2_lo;
    const float z = x * x;
    const float p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
    const float q = 1.0f + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
    const float r = p / q;
    return pio2_hi - (x - (pio2_lo - x * r));
  }
  if (hx < 0) {  // x < -0.5
    const float z = (1.0f + x) * 0.5f;
    const float p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
    const float q = 1.0f + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
    const float s = sqrtf(z);
    const float r = p / q;
    const float w = r * s - pio2_lo;
    return pi - 2.0f * (s + w);
  }
  const float z = (1.0f - x) * 0.5f;  // x > 0.5
  const float s = sqrtf(z);
  const float df = __int_as_float(__float_as_int(s) & (int)0xfffff000);
  const float c = (z - df * df) / (s + df);
  const float p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
  const float q = 1.0f + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
  const float r = p / q;
  const float w = r * s + c;
  return 2.0f * (df + w);
}

// Smallest squared distance from (px, py) to the obstacles, folded into dmin.  fminf ignores a NaN operand, so
// dmin starts as NaN ("no distance seen") and NaN distances are skipped like the reference's `minr >= r`.
__device__ __forceinline__ float dwa_min_d2(float dmin, float px, float py, const float2* ob, int n_ob) {
  for (int j = 0; j < n_ob; ++j) {
    const float dx = px - ob[j].x, dy = py - ob[j].y;
    dmin = fminf(dmin, dx * dx + dy * dy);
  }
  return dmin;
}

// calc_obstacle_cost :77-101 from the smallest squared distance over the checked points.  The reference takes
// sqrtf per pair, returns FLT_MAX at the first r <= robot_radius and otherwise keeps the minimum r.  A correctly
// rounded sqrtf is monotone, so min r = sqrtf(min d2) and "some r <= radius" is "sqrtf(min d2) <= radius": the
// same result with one square root per sample.
__device__ __forceinline__ float dwa_obstacle_cost(float dmin, float robot_radius) {
  float minr = FLT_MAX;
  if (dmin == dmin) {
    const float r = sqrtf(dmin);
    if (r <= robot_radius) return FLT_MAX;
    if (minr >= r) minr = r;
  }
  return (float)(1.0 / (double)minr);  // 1 / FLT_MAX is a float subnormal: no flush to zero anywhere here
}

// dwa_control for robot i, by the 32 lanes of its warp: the state load, the window, the sample grids in the warp's
// rows s_v / s_w, every sample's rollout and cost against the n_ob obstacles at ob (shared memory; a slice this warp
// staged itself is visible after the __syncwarp below), the argmin and the outputs.  status, when not NULL, gets
// CRB_DWA_OK.  traj gets points 0 .. n_steps; with kClip only the first max_pts of them (a traj of max_pts points
// per robot, the rest of the robot's rollout not computed).
template <bool kClip>
__device__ __forceinline__ void dwa_robot(int64_t n, int64_t i, int lane, const float2* ob, int n_ob, float* s_v,
                                          float* s_w, const float* __restrict__ xg, float* __restrict__ ug,
                                          const float* __restrict__ goalg, crb_dwa_params p, int n_steps,
                                          float* __restrict__ costg, int32_t* __restrict__ bestg,
                                          float* __restrict__ trajg, int32_t* __restrict__ statusg,
                                          int max_pts = 0) {
  float x[5];
#pragma unroll
  for (int f = 0; f < 5; ++f) x[f] = xg[(int64_t)f * n + i];
  const float gx = goalg[i], gy = goalg[n + i];
  const float u_prev1 = ug[n + i];

  // calc_dynamic_window :52-60; std::max(a, b) is (a < b) ? b : a and std::min(a, b) is (b < a) ? b : a
  const float lv = x[3] - p.max_accel * p.dt, hv = x[3] + p.max_accel * p.dt;
  const float lw = x[4] - p.max_dyawrate * p.dt, hw = x[4] + p.max_dyawrate * p.dt;
  const float dw0 = (lv < p.min_speed) ? p.min_speed : lv;
  const float dw1 = (p.max_speed < hv) ? p.max_speed : hv;
  const float dw2 = (lw < -p.max_yawrate) ? -p.max_yawrate : lw;
  const float dw3 = (p.max_yawrate < hw) ? p.max_yawrate : hw;
  // the sample grid :126-127: the k-th value is k sequential float adds (every lane runs the sequence, each
  // stores its own entries)
  int nv = 0, nw = 0;
  for (float v = dw0; nv < CRB_DWA_MAX_SPEED_SAMPLES && v <= dw1; v = v + p.v_reso, ++nv)
    if ((nv & 31) == lane) s_v[nv] = v;
  for (float w = dw2; nw < CRB_DWA_MAX_YAWRATE_SAMPLES && w <= dw3; w = w + p.yawrate_reso, ++nw)
    if ((nw & 31) == lane) s_w[nw] = w;
  __syncwarp();  // the grids (and a per-warp obstacle slice)

  const float d0 = dwa_min_d2(__int_as_float(0x7fffffff), x[0], x[1], ob, n_ob);  // point 0 is x itself
  const float gmag = sqrtf(gx * gx + gy * gy);
  float best_c = 10000.0f;  // min_cost's initial value (:120): a cost above it never wins
  int best_s = -1;
  const int ns = nv * nw;
  for (int s = lane; s < ns; s += 32) {
    const int iv = s / nw;
    const float v = s_v[iv], w = s_w[s - iv * nw];
    float st[5] = {x[0], x[1], x[2], x[3], x[4]};
    float dmin = d0;
    for (int k = 1; k <= n_steps; ++k) {  // calc_trajectory :63-74; obstacles on points 0, 2, 4, ... (:82)
      crb_dwa_motion(st, v, w, p.dt);
      if (!(k & 1)) dmin = dwa_min_d2(dmin, st[0], st[1], ob, n_ob);
    }
    // calc_to_goal_cost :103-113: std::pow(float, 2) promotes to double
    const float tmag = (float)sqrt((double)st[0] * (double)st[0] + (double)st[1] * (double)st[1]);
    const float dot = gx * st[0] + gy * st[1];
    const float to_goal = p.to_goal_cost_gain * crb_dwa_acosf(dot / (gmag * tmag));
    const float speed = p.speed_cost_gain * (p.max_speed - st[3]);
    const float cost = to_goal + speed + dwa_obstacle_cost(dmin, p.robot_radius);
    if (cost <= best_c) {  // `min_cost >= final_cost` (:136): within a lane s increases, so ties go to the later
      best_c = cost;
      best_s = s;
    }
  }
  // across lanes: the smaller cost, on a tie the larger index (= the reference's last-wins); NaN never got in
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const float oc = __shfl_xor_sync(0xffffffffu, best_c, off);
    const int os = __shfl_xor_sync(0xffffffffu, best_s, off);
    if (oc < best_c || (oc == best_c && os > best_s)) {
      best_c = oc;
      best_s = os;
    }
  }
  const int biv = best_s >= 0 ? best_s / nw : 0;
  const float bv = best_s >= 0 ? s_v[biv] : 0.0f;
  const float bw = best_s >= 0 ? s_w[best_s - biv * nw] : u_prev1;
  if (lane == 0) {
    ug[i] = bv;
    ug[n + i] = bw;
    if (costg) costg[i] = best_c;
    if (bestg) bestg[i] = best_s;
    if (statusg) statusg[i] = CRB_DWA_OK;
  }
  if (trajg) {
    const int last = kClip ? min(n_steps, max_pts - 1) : n_steps;  // the last point written
    if (best_s < 0) {
      for (int f = lane; f < 5 * (last + 1); f += 32) trajg[(int64_t)f * n + i] = __int_as_float(0x7fc00000);
    } else {
      float st[5] = {x[0], x[1], x[2], x[3], x[4]};
      for (int k = 0; k <= last; ++k) {
        if (k > 0) crb_dwa_motion(st, bv, bw, p.dt);
        if ((k & 31) == lane) {
#pragma unroll
          for (int j = 0; j < 5; ++j) trajg[(int64_t)(5 * k + j) * n + i] = st[j];
        }
      }
    }
  }
}

// ---- the parameter limits of crb.h, on the host and on the device ------------------------------------------------
static __host__ __device__ inline bool finite_pos(float v) { return isfinite(v) && v > 0.0f; }

// Spacing of binary32 values at magnitude x >= 0 (x in double; 2^-149 below the normal range).
static __host__ __device__ inline double ulp_f32(double x) {
  if (x < 0x1p-126) return 0x1p-149;
  int e = 0;
  frexp(x, &e);  // x = m 2^e, m in [0.5, 1)
  return ldexp(1.0, e - 24);
}

// Largest number of samples the reference's float loop `for (s = lo; s <= hi; s += reso)` (:126-127) can take on
// one axis, plus one, for any state.  Every sample lies in [-m, m] (the window is clipped to the limits), so each
// step s + reso rounds to at least d = reso - ulp(m + reso) / 2 above s; d <= 0 means a step can stall, and the
// result is infinite.  The window's width is at most `range` (the limits) and at most 2 fl(half) plus half an ulp
// of m for each of its rounded ends.  The extra sample of margin absorbs this function's own double rounding.
static __host__ __device__ inline double dwa_axis_samples(double m, float reso, float half, double range) {
  const double d = reso - 0.5 * ulp_f32(m + reso);
  if (!(d > 0.0)) return INFINITY;
  return fmin(2.0 * half + ulp_f32(m), range) / d + 2.0;
}

// NULL when p is inside the parameter limits of crb.h, with *n_steps = the reference's rollout step count (:67-72),
// itself bounded; otherwise the limit it breaks.  Every operation is an IEEE float or double operation (frexp, ldexp,
// fmin and fabs are exact), so the host and the device decide alike.
static __host__ __device__ inline const char* dwa_params_fault(const crb_dwa_params& p, int* n_steps) {
  if (!(isfinite(p.max_speed) && isfinite(p.min_speed) && isfinite(p.max_yawrate) && isfinite(p.max_accel) &&
        isfinite(p.robot_radius) && isfinite(p.max_dyawrate) && isfinite(p.v_reso) && isfinite(p.yawrate_reso) &&
        isfinite(p.dt) && isfinite(p.predict_time) && isfinite(p.to_goal_cost_gain) &&
        isfinite(p.speed_cost_gain)))
    return "every parameter must be finite";
  if (!(finite_pos(p.v_reso) && finite_pos(p.yawrate_reso) && finite_pos(p.dt)))
    return "v_reso, yawrate_reso and dt must be > 0";
  // the kernel's max_accel * dt and max_dyawrate * dt: a float product, formed exactly in double and rounded once
  const float hv = (float)((double)p.max_accel * p.dt), hw = (float)((double)p.max_dyawrate * p.dt);
  const double mv = fmax(fabs((double)p.min_speed), fabs((double)p.max_speed));
  if (!(dwa_axis_samples(mv, p.v_reso, hv, (double)p.max_speed - p.min_speed) <= CRB_DWA_MAX_SPEED_SAMPLES))
    return "the speed window allows more than CRB_DWA_MAX_SPEED_SAMPLES samples";
  if (!(dwa_axis_samples(fabs((double)p.max_yawrate), p.yawrate_reso, hw, 2.0 * (double)p.max_yawrate) <=
        CRB_DWA_MAX_YAWRATE_SAMPLES))
    return "the yaw-rate window allows more than CRB_DWA_MAX_YAWRATE_SAMPLES samples";
  float t = 0.0f;
  int k = 0;
  while (k <= CRB_DWA_MAX_STEPS && t <= p.predict_time) {
    t += p.dt;
    ++k;
  }
  if (!(k <= CRB_DWA_MAX_STEPS)) return "predict_time / dt allows more than CRB_DWA_MAX_STEPS rollout steps";
  *n_steps = k;
  return nullptr;
}
