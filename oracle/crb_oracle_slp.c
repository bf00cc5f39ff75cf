/* crb_oracle_slp.c — CPU restatement of sample_states, calc_uniform_polar_states, calc_biased_polar_states,
 * calc_lane_states and search_nearest_one_from_lookuptable (src/state_lattice_planner.cpp:29-135).  TEST
 * INFRASTRUCTURE ONLY (see crb_oracle.h).
 *
 * Written the way the reference is: the biased sampler fills its asi / cnav / csumnav arrays and the angle sample
 * list, sample_states then walks that list.  C's usual arithmetic conversions give every mixed float / double
 * expression the reference's types (a double literal or M_PI makes the expression double, an int operand of a float
 * expression is converted to float), the file is built with -ffp-contract=off, and sin / cos are the restatement of
 * glibc's in crb_oracle.c, never the libm of the machine this runs on.  Pinned against the reference's own text by
 * tests/test_slp.py (oracle/_ref/libref_slp.so).  The addition is CRB_SLP_OUT_OF_RANGE, for trig arguments where the
 * restated sinf / cosf are not proven.
 */
#include "crb_oracle_slp.h"

#include <float.h>
#include <math.h>
#include <stdlib.h>

#include "crb_oracle.h"

#define CRB_M_PI 3.14159265358979323846 /* M_PI of <cmath> */

typedef struct {
  float* t;
  int64_t ncol, col0;
  int k, S;
} out_t;

static void put(out_t* o, float x, float y, float yaw) {
  if (o->k >= o->S) abort(); /* S bounds every sampler's output: a violation is a bug here */
  o->t[o->col0 + o->k] = x;
  o->t[o->ncol + o->col0 + o->k] = y;
  o->t[2 * o->ncol + o->col0 + o->k] = yaw;
  o->k++;
}

static int trig_out_of_range(float a) { return fabsf(a) >= 120.0f && isfinite(a); }

/* sample_states :29-45; 0 when an angle is outside the restated sinf / cosf's range */
static int sample_states(const float* angle_samples, int n, float a_min, float a_max, int d, float p_max, float p_min,
                         int nh, out_t* o) {
  for (int s = 0; s < n; ++s) {
    const float item = angle_samples[s];
    const float a = a_min + (a_max - a_min) * item;
    if (trig_out_of_range(a)) return 0;
    for (int j = 0; j < nh; ++j) {
      float sn, cs;
      crb_oracle_libm_sincosf(a, &sn, &cs);
      const float xf = d * cs;
      const float yf = d * sn;
      float yawf;
      if (nh == 1) yawf = (p_max - p_min) / 2.0 + a;
      else yawf = p_min + (p_max - p_min) * j / (nh - 1) + a;
      put(o, xf, yf, yawf);
    }
  }
  return 1;
}

/* calc_uniform_polar_states :47-56 */
static int uniform(int nxy, int nh, int d, float a_min, float a_max, float p_min, float p_max, out_t* o) {
  float* angle_samples = (float*)malloc(sizeof(float) * (size_t)(nxy > 0 ? nxy : 1));
  for (int i = 0; i < nxy; i++) angle_samples[i] = i * 1.0 / (nxy - 1);
  const int ok = sample_states(angle_samples, nxy, a_min, a_max, d, p_max, p_min, nh, o);
  free(angle_samples);
  return ok;
}

/* calc_biased_polar_states :58-99 */
static int biased(float goal_angle, int ns, int nxy, int nh, int d, float a_min, float a_max, float p_min,
                  float p_max, out_t* o) {
  const size_t m = (size_t)(ns > 1 ? ns - 1 : 1);
  float* cnav = (float*)malloc(sizeof(float) * m);
  float* csumnav = (float*)malloc(sizeof(float) * m);
  float* angle_samples = (float*)malloc(sizeof(float) * (size_t)(nxy > 0 ? nxy : 1));
  float cnav_max = FLT_MIN;
  float cnav_sum = 0;
  for (int i = 0; i < ns - 1; i++) {
    const float asi_sample = a_min + (a_max - a_min) * i / (ns - 1);
    const float cnav_sample = CRB_M_PI - fabsf(asi_sample - goal_angle);
    cnav[i] = cnav_sample;
    cnav_sum += cnav_sample;
    if (cnav_max < cnav_sample) cnav_max = cnav_sample;
  }
  float cum_temp = 0;
  for (int i = 0; i < ns - 1; i++) {
    cnav[i] = (cnav_max - cnav[i]) / (cnav_max * ns - cnav_sum);
    cum_temp += cnav[i];
    csumnav[i] = cum_temp;
  }
  int li = 0, n = 0;
  for (int i = 0; i < nxy; i++) {
    for (int j = li; j < ns - 1; j++) {
      if (j * 1.0 / ns >= i * 1.0 / (nxy - 1)) {
        if (j < 0) abort(); /* csumnav[-1]: proven unreachable (crb_slp.cu) */
        angle_samples[n++] = csumnav[j];
        li = j - 1;
        break;
      }
    }
  }
  const int ok = sample_states(angle_samples, n, a_min, a_max, d, p_max, p_min, nh, o);
  free(cnav);
  free(csumnav);
  free(angle_samples);
  return ok;
}

/* calc_lane_states :101-113 */
static int lane(float l_center, float l_heading, float l_width, float v_width, float d, int nxy, out_t* o) {
  if (trig_out_of_range(l_heading)) return 0;
  float sn, cs;
  crb_oracle_libm_sincosf(l_heading, &sn, &cs);
  const float xc = cs * d + sn * l_center;
  const float yc = sn * d + cs * l_center;
  for (int i = 0; i < nxy; i++) {
    const float delta = -0.5 * (l_width - v_width) + (l_width - v_width) * i / (nxy - 1);
    const float xf = xc - delta * sn;
    const float yf = yc + delta * cs;
    put(o, xf, yf, l_heading);
  }
  return 1;
}

void crb_oracle_slp_sample(int64_t n_q, const crb_slp_sampler* s, int S, const float* qp, float* target,
                           int32_t* n_states, int32_t* status, int nthreads) {
  if (nthreads <= 0) nthreads = crb_oracle_num_threads();
#pragma omp parallel for num_threads(nthreads) schedule(dynamic, 64)
  for (int64_t q = 0; q < n_q; ++q) {
    out_t o = {target, n_q * S, q * S, 0, S};
    const float* f = qp + q;
    int ok;
    if (s->kind == CRB_SLP_LANE)
      ok = lane(f[0], f[n_q], f[2 * n_q], f[3 * n_q], f[4 * n_q], s->nxy, &o);
    else if (s->kind == CRB_SLP_BIASED)
      ok = biased(f[0], s->ns, s->nxy, s->nh, s->d, f[n_q], f[2 * n_q], f[3 * n_q], f[4 * n_q], &o);
    else
      ok = uniform(s->nxy, s->nh, s->d, f[0], f[n_q], f[2 * n_q], f[3 * n_q], &o);
    if (!ok) o.k = 0;
    n_states[q] = o.k;
    if (status) status[q] = ok ? CRB_SLP_OK : CRB_SLP_OUT_OF_RANGE;
    for (int j = o.k; j < S; ++j)
      for (int c = 0; c < 3; ++c) target[c * o.ncol + o.col0 + j] = NAN;
  }
}

void crb_oracle_slp_search(int64_t n, const float* target, const float* table, int rows, const float* k0,
                           float* param, int32_t* row, int nthreads) {
  if (nthreads <= 0) nthreads = crb_oracle_num_threads();
#pragma omp parallel for num_threads(nthreads) schedule(static)
  for (int64_t i = 0; i < n; ++i) {
    const float x = target[i], y = target[n + i], yaw = target[2 * n + i];
    float min_d = FLT_MAX;
    int min_id = -1;
    for (int r = 0; r < rows; r++) {
      const float* c = table + 6 * (int64_t)r;
      const float dx = x - c[0];
      const float dy = y - c[1];
      const float dyaw = yaw - c[2];
      const float d = sqrtf(dx * dx + dy * dy + dyaw * dyaw);
      if (d < min_d) {
        min_id = r;
        min_d = d;
      }
    }
    if (min_id >= 0) {
      param[i] = sqrtf(x * x + y * y);
      param[n + i] = k0 ? k0[i] : 0.0f;
      param[2 * n + i] = table[6 * (int64_t)min_id + 4];
      param[3 * n + i] = table[6 * (int64_t)min_id + 5];
    } else {
      for (int c = 0; c < 4; ++c) param[c * n + i] = NAN;
    }
    if (row) row[i] = min_id;
  }
}
