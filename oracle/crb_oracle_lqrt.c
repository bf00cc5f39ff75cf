/* crb_oracle_lqrt.c — the checker for crb_lqr_steering_control_batched and crb_lqr_update_batched (see
 * crb_oracle_lqrt.h).  The reference's text, operation for operation: float arithmetic without contraction
 * (-ffp-contract=off), the double macros DT, L and MAX_STEER promoting what they touch, YAW_P2P in double, the float
 * overloads of std::atan2 / cos / sin / tan (atan2f, cosf, sinf, tanf) and the double std::atan2 of the feed-forward. */
#define _GNU_SOURCE
#include "crb_oracle_lqrt.h"

#include <float.h>
#include <math.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "crb_oracle.h"

/* include/motion_model.h:18 YAW_P2P on a float expression, narrowed back by the assignment */
static float yaw_p2p(float a) {
  return (float)(fmod(fmod((double)a + M_PI, 2 * M_PI) - 2 * M_PI, 2 * M_PI) + M_PI);
}

float crb_oracle_lqrt_nearest(const float st[4], const float* cx, const float* cy, const float* cyaw, int32_t ncourse,
                              int32_t* ind) {
  float mind = FLT_MAX;
  for (int32_t i = 0; i < ncourse; ++i) {
    const float idx = cx[i] - st[0];
    const float idy = cy[i] - st[1];
    const float d_e = idx * idx + idy * idy;
    if (d_e < mind) {
      mind = d_e;
      *ind = i;
    }
  }
  const float dxl = cx[*ind] - st[0];
  const float dyl = cy[*ind] - st[1];
  const float angle = yaw_p2p(cyaw[*ind] - atan2f(dyl, dxl));
  if (angle < 0) mind = mind * -1;
  return mind;
}

/* solve_DARE + dlqr with crb_oracle.c's restatement, which returns the iterations executed but not whether they
 * converged: the iteration is deterministic, so a run allowed one more iteration stops within maxiter exactly when
 * this one converged (and then computes the same X and K). */
static int dlqr_conv(int nx, int nu, const float* A, const float* B, const float* Q, const float* R, int maxiter,
                     float eps, float* K, int* converged) {
  if (maxiter < 0x7fffffff) {
    const int it = crb_oracle_dlqr(nx, nu, A, B, Q, R, maxiter + 1, eps, K, NULL);
    if (it <= maxiter) {
      *converged = 1;
      return it;
    }
  }
  *converged = 0;
  return crb_oracle_dlqr(nx, nu, A, B, Q, R, maxiter, eps, K, NULL);
}

/* lqr_steering_control :98-133 (nx 4) / :108-151 (nx 5) for vehicle i */
static void control_one(int64_t n, int64_t i, int nx, const float* state, const float* cx, const float* cy,
                        const float* cyaw, const float* ck, const float* sp, int32_t ncourse,
                        const crb_oracle_lqrt_params* p, int32_t* ind, float* pe, float* pth_e, float* u, float* K,
                        int32_t* iters, int32_t* status) {
  const int nu = nx == 4 ? 1 : 2;
  const float st[4] = {state[i], state[n + i], state[2 * n + i], state[3 * n + i]};
  int32_t j = nx == 4 ? ind[i] : 0;
  /* the scan first, on its own, to learn whether the reference would read out of bounds */
  float mind = FLT_MAX;
  int won = 0;
  for (int32_t c = 0; c < ncourse; ++c) {
    const float idx = cx[c] - st[0], idy = cy[c] - st[1];
    const float d_e = idx * idx + idy * idy;
    if (d_e < mind) { mind = d_e; won = 1; }
  }
  if (!won && (j < 0 || j >= ncourse)) {
    for (int r = 0; r < nu; ++r) u[(int64_t)r * n + i] = NAN;
    if (K) for (int f = 0; f < nu * nx; ++f) K[(int64_t)f * n + i] = NAN;
    if (iters) iters[i] = 0;
    if (status) status[i] = 2;
    return;
  }
  const float e = crb_oracle_lqrt_nearest(st, cx, cy, cyaw, ncourse, &j);
  const double DT = p->dt, L = p->wheelbase;
  const float k = ck[j];
  const float th_e = yaw_p2p(st[2] - cyaw[j]);
  float A[25] = {0}, B[10] = {0}, Q[25], R[4], Kk[10];
  A[0 + nx * 0] = 1.0f;
  A[0 + nx * 1] = (float)DT;
  A[1 + nx * 2] = st[3];
  A[2 + nx * 2] = 1.0f;
  A[2 + nx * 3] = (float)DT;
  B[3] = (float)(st[3] / L);
  if (nx == 5) {
    A[4 + nx * 4] = 1.0f;
    B[4 + nx * 1] = (float)DT;
  }
  for (int r = 0; r < nx; ++r) for (int c = 0; c < nx; ++c) Q[r + nx * c] = p->Q[r + 5 * c];
  for (int r = 0; r < nu; ++r) for (int c = 0; c < nu; ++c) R[r + nu * c] = p->R[r + 2 * c];
  int conv;
  const int it = dlqr_conv(nx, nu, A, B, Q, R, p->maxiter, p->eps, Kk, &conv);
  float x[5];
  x[0] = e;
  x[1] = (float)((e - pe[i]) / DT);
  x[2] = th_e;
  x[3] = (float)((th_e - pth_e[i]) / DT);
  if (nx == 5) x[4] = st[3] - sp[j];
  float us[2];
  for (int r = 0; r < nu; ++r) {  /* (-K) * x: Eigen's unary minus, then the product */
    float s = (-Kk[r]) * x[0];
    for (int c = 1; c < nx; ++c) s = s + (-Kk[r + nu * c]) * x[c];
    us[r] = s;
  }
  const float ff = (float)atan2(L * k, (double)1.0);
  const float fb = yaw_p2p(us[0]);
  const float delta = ff + fb;
  if (nx == 4) {
    u[i] = delta;
  } else {
    u[i] = us[1];
    u[n + i] = delta;
  }
  ind[i] = j;
  pe[i] = e;
  pth_e[i] = th_e;
  if (K) for (int f = 0; f < nu * nx; ++f) K[(int64_t)f * n + i] = Kk[f];
  if (iters) iters[i] = it;
  if (status) status[i] = conv ? 0 : 1;
}

void crb_oracle_lqrt_control_batched(int64_t n, int nx, const float* state, const float* cx, const float* cy,
                                     const float* cyaw, const float* ck, const float* sp, int32_t ncourse,
                                     const crb_oracle_lqrt_params* p, int32_t* ind, float* pe, float* pth_e, float* u,
                                     float* K, int32_t* iters, int32_t* status, int nthreads) {
#ifdef _OPENMP
  if (nthreads <= 0) nthreads = omp_get_max_threads();
#pragma omp parallel for num_threads(nthreads) schedule(dynamic, 64)
#endif
  for (int64_t i = 0; i < n; ++i)
    control_one(n, i, nx, state, cx, cy, cyaw, ck, sp, ncourse, p, ind, pe, pth_e, u, K, iters, status);
  (void)nthreads;
}

/* update :136-146 / :154-164 */
void crb_oracle_lqrt_update_batched(int64_t n, float* state, const float* a, const float* delta,
                                    const crb_oracle_lqrt_params* p, int nthreads) {
#ifdef _OPENMP
  if (nthreads <= 0) nthreads = omp_get_max_threads();
#pragma omp parallel for num_threads(nthreads) schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i) {
    const double MAX_STEER = p->max_steer, DT = p->dt, L = p->wheelbase;
    float d = delta[i];
    if (d >= MAX_STEER) d = MAX_STEER;
    if (d <= -MAX_STEER) d = -MAX_STEER;
    float x = state[i], y = state[n + i], yaw = state[2 * n + i], v = state[3 * n + i];
    const float nx = x + v * cosf(yaw) * DT;
    const float ny = y + v * sinf(yaw) * DT;
    const float nyaw = yaw + v / L * tanf(d) * DT;
    const float nv = v + a[i] * DT;
    state[i] = nx; state[n + i] = ny; state[2 * n + i] = nyaw; state[3 * n + i] = nv;
  }
  (void)nthreads;
}

int64_t crb_oracle_lqrt_ff_check(double L, uint32_t lo_bits, uint32_t hi_bits, const float* got) {
  int64_t bad = 0;
#ifdef _OPENMP
#pragma omp parallel for reduction(+ : bad) schedule(static, 65536)
#endif
  for (int64_t b = lo_bits; b < (int64_t)hi_bits; ++b) {
    const uint32_t u = (uint32_t)b;
    float k;
    memcpy(&k, &u, 4);
    const float want = (float)atan2(L * k, (double)1.0);
    if (memcmp(&want, &got[b - lo_bits], 4) != 0) ++bad;
  }
  return bad;
}
