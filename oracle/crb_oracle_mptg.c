/* crb_oracle_mptg.c — CPU restatement of TrajectoryOptimizer::optimizer_traj (include/trajectory_optimizer.h
 * :53-200) and MotionModel (include/motion_model.h:59-150).  TEST INFRASTRUCTURE ONLY (see crb_oracle.h).
 *
 * Written the way the reference is: every iteration rolls the nominal parameter out again and keeps its points
 * (:64), the Jacobian takes six generate_last_state calls (:146-175), the line search two (:178-200), and the
 * returned Traj is the last nominal.  Every float operation is separately rounded (built -ffp-contract=off),
 * YAW_P2P and the cost are in double, the 3x3 inverses are Eigen 3.3's cofactor formula, and sinf / cosf / tanf
 * are restatements of glibc's, never the libm of the machine this runs on.  Pinned against the reference's own
 * text by tests/test_mptg.py (oracle/_ref/libref_mptg.so).  The additions are include/crb.h's statuses, for the
 * cases the reference leaves undefined or where the restated tanf / sinf / cosf are not proven.
 */
#include "crb_oracle_mptg.h"

#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "crb_oracle.h"

#define CRB_M_PI 3.14159265358979323846 /* M_PI of <cmath> */

static uint32_t bits_of(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
}
static float float_of(uint32_t u) {
  float f;
  memcpy(&f, &u, 4);
  return f;
}

/* ---- glibc 2.39's tanf ----------------------------------------------------------------------------------
 * sysdeps/ieee754/flt-32/s_tanf.c + k_tanf.c (fdlibm, Sun Microsystems, freely redistributable) with
 * e_rem_pio2f.c's binary64 reduce_fast (x - n * pi/2 is a separate multiply and subtract: that file is not built
 * with FMA, unlike s_sinf.c).  |x| >= 120 (reduce_large) is not restated. */
static float kernel_tanf(float x, float y, int iy) {
  static const float T[] = {3.3333334327e-01f, 1.3333334029e-01f, 5.3968254477e-02f, 2.1869488060e-02f,
                            8.8632395491e-03f, 3.5920790397e-03f, 1.4562094584e-03f, 5.8804126456e-04f,
                            2.4646313977e-04f, 7.8179444245e-05f, 7.1407252108e-05f, -1.8558637748e-05f,
                            2.5907305826e-05f};
  const float pio4 = 7.8539812565e-01f, pio4lo = 3.7748947079e-08f;
  float z, r, v, w, s;
  const int32_t hx = (int32_t)bits_of(x);
  const int32_t ix = hx & 0x7fffffff;
  if (ix < 0x39000000) { /* |x| < 2^-13: (int)x == 0 */
    if ((ix | (iy + 1)) == 0) return 1.0f / fabsf(x);
    if (iy == 1) return x;
    return -1.0f / x;
  }
  if (ix >= 0x3f2ca140) { /* |x| >= 0.6744 */
    if (hx < 0) {
      x = -x;
      y = -y;
    }
    z = pio4 - x;
    w = pio4lo - y;
    x = z + w;
    y = 0.0f;
    if (fabsf(x) < 0x1p-13f) return (1 - ((hx >> 30) & 2)) * iy * (1.0f - 2 * iy * x);
  }
  z = x * x;
  w = z * z;
  r = T[1] + w * (T[3] + w * (T[5] + w * (T[7] + w * (T[9] + w * T[11]))));
  v = z * (T[2] + w * (T[4] + w * (T[6] + w * (T[8] + w * (T[10] + w * T[12])))));
  s = z * x;
  r = y + z * (s * (r + v) + y);
  r += T[0] * s;
  w = x + r;
  if (ix >= 0x3f2ca140) {
    v = (float)iy;
    return (float)(1 - ((hx >> 30) & 2)) * (v - 2.0f * (x - (w * w / (w + v) - r)));
  }
  if (iy == 1) return w;
  {
    float a, t;
    z = float_of(bits_of(w) & 0xfffff000u);
    v = r - (z - x);
    t = a = -1.0f / w;
    t = float_of(bits_of(t) & 0xfffff000u);
    s = 1.0f + t * z;
    return t + a * (s + t * v);
  }
}

float crb_oracle_libm_tanf(float x) {
  const uint32_t ix = bits_of(x) & 0x7fffffffu;
  if (ix <= 0x3f490fdau) return kernel_tanf(x, 0.0f, 1);
  if (ix >= 0x7f800000u) return x - x;
  if (ix >= 0x42f00000u) return NAN; /* |x| >= 120: not restated (callers stop before) */
  const double dx = x;
  const double r = dx * 0x1.45F306DC9C883p+23;
  const int n = ((int32_t)r + 0x800000) >> 24;
  const double prod = (double)n * 0x1.921FB54442D18p0;
  const double d = dx - prod;
  const float y0 = (float)d;
  const float y1 = (float)(d - y0);
  return kernel_tanf(y0, y1, 1 - ((n & 1) << 1));
}

int64_t crb_oracle_libm_tanf_census(uint32_t lo_bits, uint32_t hi_bits) {
  int64_t bad = 0;
#pragma omp parallel for reduction(+ : bad) schedule(static, 1 << 16)
  for (int64_t u = lo_bits; u < (int64_t)hi_bits; ++u) {
    for (int sg = 0; sg < 2; ++sg) {
      const float y = float_of((uint32_t)u | (sg ? 0x80000000u : 0u));
      volatile float h = tanf(y);
      const float hv = h, m = crb_oracle_libm_tanf(y);
      bad += memcmp(&hv, &m, 4) != 0 && !(isnan(hv) && isnan(m));
    }
  }
  return bad;
}

int64_t crb_oracle_libm_tanf_check(uint32_t lo_bits, uint32_t hi_bits, const float* got) {
  int64_t bad = 0;
#pragma omp parallel for reduction(+ : bad) schedule(static, 1 << 16)
  for (int64_t u = lo_bits; u < (int64_t)hi_bits; ++u) {
    for (int sg = 0; sg < 2; ++sg) {
      const float m = crb_oracle_libm_tanf(float_of((uint32_t)u | (sg ? 0x80000000u : 0u)));
      const float g = got[2 * (u - lo_bits) + sg];
      bad += memcmp(&g, &m, 4) != 0 && !(isnan(g) && isnan(m));
    }
  }
  return bad;
}

/* ---- include/motion_model.h ------------------------------------------------------------------------------ */
typedef struct {
  float x, y, yaw;
} traj_state;

/* YAW_P2P :18 on a float argument, assigned back to float */
static float yaw_p2p(float angle) {
  return (float)(fmod(fmod((double)angle + CRB_M_PI, 2 * CRB_M_PI) - 2 * CRB_M_PI, 2 * CRB_M_PI) + CRB_M_PI);
}

/* Eigen 3.3's compute_inverse<Matrix3f, Matrix3f, 3> (m[r][c]), then the product with y in k order; returns
 * whether every entry of the inverse is finite */
static float cofactor(const float m[3][3], int i, int j) {
  const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
  return m[i1][j1] * m[i2][j2] - m[i1][j2] * m[i2][j1];
}
static int inverse_times(const float m[3][3], const float y[3], float out[3]) {
  float c[3], inv[3][3];
  for (int i = 0; i < 3; ++i) c[i] = cofactor(m, i, 0);
  const float det = c[0] * m[0][0] + c[1] * m[1][0] + c[2] * m[2][0];
  const float invdet = 1.0f / det;
  int finite = 1;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      inv[i][j] = (i == 0 ? c[j] : cofactor(m, j, i)) * invdet;
      finite &= isfinite(inv[i][j]) != 0;
    }
  for (int i = 0; i < 3; ++i) out[i] = inv[i][0] * y[0] + inv[i][1] * y[1] + inv[i][2] * y[2];
  return finite;
}

typedef struct {
  float x, y, yaw, v;
} state4;

/* generate_trajectory :110-131 (points to out[] when given, at most max_out of them) and generate_last_state
 * :133-150 (*last).  Returns 0, CRB_MPTG_STEP_CAP or CRB_MPTG_OUT_OF_RANGE; *steps is the number of points. */
static int rollout(const state4* st0, const crb_mptg_params* c, float distance, const float steer[3],
                   traj_state* out, int max_out, traj_state* last, int* steps, int* quirks) {
  const float n = distance / c->ds;
  const float horizon = distance / st0->v;
  /* quadratic_interpolation({0, horizon/2, horizon}, steering) :59-72 */
  const float xs[3] = {0.0f, horizon / 2, horizon};
  float A[3][3], spline[3];
  for (int r = 0; r < 3; ++r) {
    A[r][0] = (float)pow(xs[r], 2);
    A[r][1] = xs[r];
    A[r][2] = 1.0f;
  }
  inverse_times(A, steer, spline);
  state4 s = *st0;
  int k = 0, rc = 0;
  for (float i = 0.0f; i < horizon; i += horizon / n) {
    if (k == CRB_MPTG_MAX_STEPS) {
      rc = CRB_MPTG_STEP_CAP;
      break;
    }
    const float kp = spline[0] * i * i + spline[1] * i + spline[2]; /* interp_refer :74-76 */
    if (fabsf(kp) >= 120.0f && isfinite(kp)) {
      rc = CRB_MPTG_OUT_OF_RANGE;
      break;
    }
    if (quirks && fabsf(kp) > 7.8539816e-01f) *quirks |= CRB_ORACLE_MPTG_STEER_BEYOND_PIO4;
    /* MotionModel::update(State, delta, dt) :102-108 */
    const float dt = horizon / n;
    float sn, cs;
    crb_oracle_libm_sincosf(s.yaw, &sn, &cs);
    s.x = s.x + s.v * cs * dt;
    s.y = s.y + s.v * sn * dt;
    s.yaw = s.yaw + s.v / c->base_l * crb_oracle_libm_tanf(kp) * dt;
    s.yaw = yaw_p2p(s.yaw);
    if (out && k < max_out) {
      out[k].x = s.x;
      out[k].y = s.y;
      out[k].yaw = s.yaw;
    }
    ++k;
  }
  *steps = k;
  last->x = s.x;
  last->y = s.y;
  last->yaw = s.yaw;
  return rc;
}

/* calc_diff :130-135 and the cost of :108-109 / :191 */
static float diff_cost(const float tg[3], const traj_state* ls, float dc[3]) {
  dc[0] = tg[0] - ls->x;
  dc[1] = tg[1] - ls->y;
  const float yaw_ = tg[2] - ls->yaw;
  dc[2] = yaw_p2p(yaw_);
  return (float)sqrt(pow(dc[0], 2) + pow(dc[1], 2) + pow(dc[2], 2));
}

/* the worse of two group statuses: OUT_OF_RANGE before STEP_CAP (the kernel's rule) */
static int worse(int a, int b) {
  if (a == CRB_MPTG_OUT_OF_RANGE || b == CRB_MPTG_OUT_OF_RANGE) return CRB_MPTG_OUT_OF_RANGE;
  return a ? a : b;
}

static void optimize_one(int64_t n, int64_t i, const float* stg, const float* tgg, float* pg,
                         const crb_mptg_params* c, int max_pts, float* traj, int32_t* traj_len, float* cost,
                         int32_t* status, int32_t* iters, int32_t* quirks, traj_state* buf) {
  const state4 st = {stg[i], stg[n + i], stg[2 * n + i], stg[3 * n + i]};
  const float tg[3] = {tgg[i], tgg[n + i], tgg[2 * n + i]};
  float dist = pg[i];
  float steer[3] = {pg[n + i], pg[2 * n + i], pg[3 * n + i]};
  int stat = CRB_MPTG_MAX_ITER_REACHED, count = 0, q = 0, len = 0;
  float out_cost = NAN;
  if (!(fabsf(st.yaw) < 120.0f)) stat = CRB_MPTG_OUT_OF_RANGE;
  for (int it = 0; stat == CRB_MPTG_MAX_ITER_REACHED && it < c->max_iter; ++it) {
    /* sample_traj = generate_trajectory(p) :64 */
    traj_state last;
    int steps = 0;
    int rc = rollout(&st, c, dist, steer, buf, max_pts, &last, &steps, &q);
    if (rc) {
      stat = rc;
      break;
    }
    if (steps == 0) {
      stat = CRB_MPTG_EMPTY_TRAJ;
      break;
    }
    if ((double)steps != ceil((double)(dist / c->ds))) q |= CRB_ORACLE_MPTG_STEPS_OFF_CEIL;
    len = steps;
    float dc[3];
    const float cst = diff_cost(tg, &last, dc);
    out_cost = cst;
    if (cst < c->cost_th) {
      stat = CRB_MPTG_CONVERGED;
      if (it == 0) q |= CRB_ORACLE_MPTG_CONVERGED_AT_0;
      break;
    }
    /* calc_J :146-175 */
    float J[3][3];
    for (int col = 0; col < 3; ++col) { /* all six roll-outs: the group's status does not depend on their order */
      const float h = c->h_step[col];
      float ev[2][3];
      for (int sg = 0; sg < 2; ++sg) {
        float d2 = dist, s2[3] = {steer[0], steer[1], steer[2]};
        if (col == 0) d2 = sg ? dist - h : dist + h;
        else s2[col] = sg ? steer[col] - h : steer[col] + h;
        traj_state ls;
        int k2;
        rc = worse(rc, rollout(&st, c, d2, s2, NULL, 0, &ls, &k2, &q));
        diff_cost(tg, &ls, ev[sg]);
      }
      for (int r = 0; r < 3; ++r) J[r][col] = (ev[0][r] - ev[1][r]) / (float)(2.0 * h);
    }
    if (rc) {
      stat = rc;
      break;
    }
    float dp[3];
    if (!inverse_times(J, dc, dp)) q |= CRB_ORACLE_MPTG_SINGULAR_J;
    for (int k = 0; k < 3; ++k) dp[k] = -dp[k];
    /* selection_learning_param :178-200 */
    float mincost = FLT_MAX, mina = 1.0f, lc[2];
    int ia = 0;
    for (float a = 1.0f; a < 2.0f; a += 0.5f, ++ia) {
      float d2 = dist, s2[3] = {steer[0], steer[1], steer[2]};
      d2 += a * dp[0];
      s2[1] += a * dp[1];
      s2[2] += a * dp[2];
      traj_state ls;
      int k2;
      rc = worse(rc, rollout(&st, c, d2, s2, NULL, 0, &ls, &k2, &q));
      float dd[3];
      const float cc = diff_cost(tg, &ls, dd);
      lc[ia] = cc;
      if ((cc <= mincost) && (a != 0.0f)) {
        mina = a;
        mincost = cc;
      }
    }
    if (rc) {
      stat = rc;
      break;
    }
    if (isnan(lc[0]) || isnan(lc[1])) q |= CRB_ORACLE_MPTG_LS_NAN;
    if (lc[0] == lc[1] && lc[0] <= FLT_MAX) q |= CRB_ORACLE_MPTG_LS_TIE;
    dist += mina * dp[0];
    steer[1] += mina * dp[1];
    steer[2] += mina * dp[2];
    count++;
  }
  const int has_traj = stat == CRB_MPTG_CONVERGED || stat == CRB_MPTG_MAX_ITER_REACHED;
  if (!has_traj) {
    len = 0;
    out_cost = NAN;
  }
  pg[i] = dist;
  for (int k = 0; k < 3; ++k) pg[(k + 1) * n + i] = steer[k];
  if (traj_len) traj_len[i] = len;
  if (cost) cost[i] = out_cost;
  if (status) status[i] = stat;
  if (iters) iters[i] = count;
  if (quirks) quirks[i] = q;
  if (traj)
    for (int k = 0; k < len && k < max_pts; ++k) {
      traj[(3 * (int64_t)k) * n + i] = buf[k].x;
      traj[(3 * (int64_t)k + 1) * n + i] = buf[k].y;
      traj[(3 * (int64_t)k + 2) * n + i] = buf[k].yaw;
    }
}

void crb_oracle_mptg_optimize(int64_t n, const float* state, const float* target, float* param,
                              const crb_mptg_params* p, int max_pts, float* traj, int32_t* traj_len, float* cost,
                              int32_t* status, int32_t* iters, int32_t* quirks, int nthreads) {
  if (nthreads <= 0) nthreads = crb_oracle_num_threads();
#pragma omp parallel num_threads(nthreads)
  {
    traj_state* buf = (traj_state*)malloc(sizeof(traj_state) * (size_t)(max_pts > 0 ? max_pts : 1));
#pragma omp for schedule(dynamic, 16)
    for (int64_t i = 0; i < n; ++i)
      optimize_one(n, i, state, target, param, p, max_pts, traj, traj_len, cost, status, iters, quirks, buf);
    free(buf);
  }
}

void crb_oracle_mptg_generate(int64_t n, const float* state, const float* param, const crb_mptg_params* p,
                              int max_pts, float* traj, int32_t* traj_len, float* last, int32_t* status,
                              int nthreads) {
  if (nthreads <= 0) nthreads = crb_oracle_num_threads();
#pragma omp parallel num_threads(nthreads)
  {
    traj_state* buf = (traj_state*)malloc(sizeof(traj_state) * (size_t)(max_pts > 0 ? max_pts : 1));
#pragma omp for schedule(dynamic, 16)
    for (int64_t i = 0; i < n; ++i) {
      const state4 st = {state[i], state[n + i], state[2 * n + i], state[3 * n + i]};
      const float steer[3] = {param[n + i], param[2 * n + i], param[3 * n + i]};
      traj_state ls;
      int k = 0, rc = CRB_MPTG_OUT_OF_RANGE;
      if (fabsf(st.yaw) < 120.0f) rc = rollout(&st, p, param[i], steer, buf, max_pts, &ls, &k, NULL);
      if (rc) {
        k = 0;
        ls.x = ls.y = ls.yaw = NAN;
      }
      if (traj_len) traj_len[i] = k;
      if (status) status[i] = rc;
      if (last) {
        last[i] = ls.x;
        last[n + i] = ls.y;
        last[2 * n + i] = ls.yaw;
      }
      if (traj)
        for (int j = 0; j < k && j < max_pts; ++j) {
          traj[(3 * (int64_t)j) * n + i] = buf[j].x;
          traj[(3 * (int64_t)j + 1) * n + i] = buf[j].y;
          traj[(3 * (int64_t)j + 2) * n + i] = buf[j].yaw;
        }
    }
    free(buf);
  }
}
