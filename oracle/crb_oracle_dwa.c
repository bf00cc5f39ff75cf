/* crb_oracle_dwa.c — CPU restatement of src/dynamic_window_approach.cpp (motion :43-50, dwa_control :148-155).
 * TEST INFRASTRUCTURE ONLY (see crb_oracle.h).
 *
 * Written the way the reference is: per sample the whole trajectory (:63-74), the obstacle cost with one
 * sqrtf per (point, obstacle) pair and the early return (:77-101), the goal cost with std::pow promoted to
 * double (:103-113) and the `min_cost >= final_cost` scan in v-major order (:120-143).  Pinned against the
 * reference's own text by tests/test_dwa.py (oracle/_ref/libref_dwa.so).  The only additions are the caps of
 * include/crb.h on the sample grid and the rollout length, where the reference's loops would not end.
 */
#include "crb_oracle_dwa.h"

#include <float.h>
#include <math.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "crb_oracle.h"

/* glibc 2.39's acosf: fdlibm's binary32 e_acosf.c (Sun Microsystems, freely redistributable), restated. */
float crb_oracle_libm_acosf(float x) {
  const float pi = 3.1415925026e+00f, pio2_hi = 1.5707962513e+00f, pio2_lo = 7.5497894159e-08f;
  const float pS0 = 1.6666667163e-01f, pS1 = -3.2556581497e-01f, pS2 = 2.0121252537e-01f,
              pS3 = -4.0055535734e-02f, pS4 = 7.9153501429e-04f, pS5 = 3.4793309169e-05f;
  const float qS1 = -2.4033949375e+00f, qS2 = 2.0209457874e+00f, qS3 = -6.8828397989e-01f,
              qS4 = 7.7038154006e-02f;
  int32_t hx;
  memcpy(&hx, &x, 4);
  const int32_t ix = hx & 0x7fffffff;
  if (ix == 0x3f800000) return hx > 0 ? 0.0f : pi + 2.0f * pio2_lo;
  if (ix > 0x3f800000) return (x - x) / (x - x);
  if (ix < 0x3f000000) {
    if (ix <= 0x23000000) return pio2_hi + pio2_lo;
    const float z = x * x;
    const float p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
    const float q = 1.0f + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
    const float r = p / q;
    return pio2_hi - (x - (pio2_lo - x * r));
  }
  if (hx < 0) {
    const float z = (1.0f + x) * 0.5f;
    const float p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
    const float q = 1.0f + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
    const float s = sqrtf(z);
    const float r = p / q;
    const float w = r * s - pio2_lo;
    return pi - 2.0f * (s + w);
  }
  const float z = (1.0f - x) * 0.5f;
  const float s = sqrtf(z);
  float df = s;
  int32_t idf;
  memcpy(&idf, &df, 4);
  idf &= (int32_t)0xfffff000;
  memcpy(&df, &idf, 4);
  const float c = (z - df * df) / (s + df);
  const float p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
  const float q = 1.0f + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
  const float r = p / q;
  const float w = r * s + c;
  return 2.0f * (df + w);
}

int64_t crb_oracle_libm_acosf_census(uint32_t lo_bits, uint32_t hi_bits) {
  int64_t bad = 0;
#pragma omp parallel for reduction(+ : bad) schedule(static)
  for (int64_t u = lo_bits; u < (int64_t)hi_bits; ++u) {
    const uint32_t b = (uint32_t)u;
    for (int sg = 0; sg < 2; ++sg) {
      const uint32_t bs = b | (sg ? 0x80000000u : 0u);
      float y;
      memcpy(&y, &bs, 4);
      volatile float h = acosf(y);
      const float hv = h, m = crb_oracle_libm_acosf(y);
      bad += memcmp(&hv, &m, 4) != 0;
    }
  }
  return bad;
}

/* motion :43-50 with glibc's sinf / cosf (restated in crb_oracle.c, bitwise the host libm for |yaw| < 120) */
static void motion(float s[5], float v, float w, float dt) {
  s[2] += w * dt;
  float sn, cs;
  crb_oracle_libm_sincosf(s[2], &sn, &cs);
  s[0] += v * cs * dt;
  s[1] += v * sn * dt;
  s[3] = v;
  s[4] = w;
}

void crb_oracle_dwa_motion(int64_t n, float* x, const float* u, float dt, int nthreads) {
  if (nthreads <= 0) nthreads = crb_oracle_num_threads();
#pragma omp parallel for num_threads(nthreads) schedule(static)
  for (int64_t i = 0; i < n; ++i) {
    float s[5];
    for (int f = 0; f < 5; ++f) s[f] = x[f * n + i];
    motion(s, u[i], u[n + i], dt);
    for (int f = 0; f < 5; ++f) x[f * n + i] = s[f];
  }
}

/* calc_trajectory :63-74 into tr (5 floats per point); returns the number of points */
static int trajectory(const float x0[5], float v, float w, const crb_dwa_params* c, float* tr) {
  float s[5];
  memcpy(s, x0, sizeof(s));
  memcpy(tr, s, sizeof(s));
  int np = 1;
  float time = 0.0f;
  while (time <= c->predict_time && np <= CRB_DWA_MAX_STEPS) {
    motion(s, v, w, c->dt);
    memcpy(tr + 5 * np++, s, sizeof(s));
    time += c->dt;
  }
  return np;
}

/* calc_obstacle_cost :77-101 */
static float obstacle_cost(const float* tr, int np, const float* ob, int n_ob, const crb_dwa_params* c) {
  float minr = FLT_MAX;
  for (int ii = 0; ii < np; ii += 2) {
    for (int k = 0; k < n_ob; ++k) {
      const float dx = tr[5 * ii] - ob[2 * k], dy = tr[5 * ii + 1] - ob[2 * k + 1];
      const float r = sqrtf(dx * dx + dy * dy);
      if (r <= c->robot_radius) return FLT_MAX;
      if (minr >= r) minr = r;
    }
  }
  return (float)(1.0 / minr);
}

/* calc_to_goal_cost :103-113 */
static float to_goal_cost(const float* last, float gx, float gy, const crb_dwa_params* c) {
  const float goal_magnitude = sqrtf(gx * gx + gy * gy);
  const float traj_magnitude = (float)sqrt(pow((double)last[0], 2) + pow((double)last[1], 2));
  const float dot_product = (gx * last[0]) + (gy * last[1]);
  const float error = dot_product / (goal_magnitude * traj_magnitude);
  return c->to_goal_cost_gain * crb_oracle_libm_acosf(error);
}

static void dwa_one(int64_t n, int64_t i, const float* xg, float* ug, const float* goal, const float* ob,
                    int n_ob, const crb_dwa_params* c, float* cost, int32_t* best, float* traj, float* tr) {
  float x[5];
  for (int f = 0; f < 5; ++f) x[f] = xg[f * n + i];
  const float gx = goal[i], gy = goal[n + i];
  /* calc_dynamic_window :52-60 (std::max / std::min) */
  const float a0 = x[3] - c->max_accel * c->dt, a1 = x[3] + c->max_accel * c->dt;
  const float a2 = x[4] - c->max_dyawrate * c->dt, a3 = x[4] + c->max_dyawrate * c->dt;
  const float dw0 = (a0 < c->min_speed) ? c->min_speed : a0;
  const float dw1 = (c->max_speed < a1) ? c->max_speed : a1;
  const float dw2 = (a2 < -c->max_yawrate) ? -c->max_yawrate : a2;
  const float dw3 = (c->max_yawrate < a3) ? c->max_yawrate : a3;
  /* calc_final_input :115-145 */
  float min_cost = 10000.0f;
  float mu0 = 0.0f, mu1 = ug[n + i];
  int32_t bs = -1, s = 0;
  int iv = 0;
  for (float v = dw0; iv < CRB_DWA_MAX_SPEED_SAMPLES && v <= dw1; v += c->v_reso, ++iv) {
    int iw = 0;
    for (float y = dw2; iw < CRB_DWA_MAX_YAWRATE_SAMPLES && y <= dw3; y += c->yawrate_reso, ++iw, ++s) {
      const int np = trajectory(x, v, y, c, tr);
      const float* last = tr + 5 * (np - 1);
      const float tg = to_goal_cost(last, gx, gy, c);
      const float sp = c->speed_cost_gain * (c->max_speed - last[3]);
      const float oc = obstacle_cost(tr, np, ob, n_ob, c);
      const float final_cost = tg + sp + oc;
      if (min_cost >= final_cost) {
        min_cost = final_cost;
        mu0 = v;
        mu1 = y;
        bs = s;
      }
    }
  }
  ug[i] = mu0;
  ug[n + i] = mu1;
  if (cost) cost[i] = min_cost;
  if (best) best[i] = bs;
  if (traj) { /* best_traj; the reference returns an empty Traj when nothing is admissible: NaN here */
    const int np = trajectory(x, mu0, mu1, c, tr);
    for (int k = 0; k < np; ++k)
      for (int j = 0; j < 5; ++j) traj[(5 * k + j) * n + i] = bs >= 0 ? tr[5 * k + j] : NAN;
  }
}

void crb_oracle_dwa_control(int64_t n, const float* x, float* u, const float* goal, const float* ob, int n_ob,
                            const crb_dwa_params* c, float* cost, int32_t* best, float* traj, int nthreads) {
  if (nthreads <= 0) nthreads = crb_oracle_num_threads();
#pragma omp parallel num_threads(nthreads)
  {
    float tr[5 * (CRB_DWA_MAX_STEPS + 2)]; /* one trajectory per thread */
#pragma omp for schedule(dynamic, 16)
    for (int64_t i = 0; i < n; ++i) dwa_one(n, i, x, u, goal, ob, n_ob, c, cost, best, traj, tr);
  }
}
