/* crb_oracle_mpc.c — CPU restatement of the MPC path.  TEST INFRASTRUCTURE ONLY.
 *
 * PROBLEM (restated from the reference, pinned against its own FG_EVAL source compiled with a CppAD
 * shim, see oracle/shim): src/model_predictive_control.cpp
 *   variables / layout   :54-60      cost   :202-210, :247-250      dynamics  :242-245
 *   bounds  :283-301      cold start :266-274   plant step update() :69-81
 *   calc_nearest_index :107-127      calc_ref_trajectory :130-170
 *
 * SOLVER (PARITY UNPINNED against the reference: the reference hands the NLP to CppAD + IPOPT
 * (:334-336), third-party code that is not in /root/reference, not installed here, and is stopped by
 * a CPU-time limit (:328), so its output is not reproducible even on its own machine).  BASELINE.json's
 * north_star replaces it by "horizon-T linearised dynamics, QP cost, Riccati factorise-and-solve";
 * this file is the executable specification of that replacement, and libcrb's kernel must match it
 * BIT FOR BIT.  Its fixed point is the KKT point of the reference NLP, which tests/ checks against
 * SciPy SLSQP on the exact NLP and against the independent float64 statement in tests/ref_mpc.py.
 *
 *   repeat (at most max_iter times; IPOPT's own cap is 50, :326)
 *     backward sweep t = T-2..0 along the current roll-out (X, U):
 *       linearise the dynamics (A_t, B_t and their second derivatives), build the quadratic model of
 *       the cost-to-go in (x_t, w_t = u_{t-1}, u_t)   [w carries the input-rate cost :207-210],
 *       projected-Newton step of the 2-D box QP in u_t (Quu may be indefinite: inputs pinned to a bound
 *       by the gradient are fixed, the Hessian of the others is shifted to positive definite)
 *       (|delta| <= MAX_STEER, |a| <= MAX_ACCEL, MIN_SPEED <= v_{t+1} <= MAX_SPEED folded into the
 *       bound on a_t), feedback gains for the free inputs, Riccati update of the value function
 *     forward sweep with step alpha = 1, 1/2, ... : clamped non-linear roll-out under the affine
 *       policy; accept the first alpha that decreases the cost (difference accumulated term by term
 *       as (q'-q)(q'+q) so that it is accurate in binary32)
 *     (if no alpha decreases the cost, the sweep is redone once in Gauss-Newton mode, i.e. without the
 *      second-derivative terms, which always yields a descent direction)
 *   until sum|dU| <= du_th, or the full step changes the cost by <= j_tol * cost (binary32 cannot
 *   resolve more), or neither mode decreases the cost
 *
 * ARITHMETIC CONTRACT shared with the CUDA kernel: binary32 throughout; every a*b+c that is meant
 * to be fused is written fmaf(); nothing else may be contracted (gcc -ffp-contract=off, nvcc
 * -fmad=false); sums run in ascending index order starting from the first product; sin/cos are the
 * polynomial crb_sincosf below (not libm); '/', sqrtf and rintf are IEEE-exact on both sides; 1/dt and
 * 1/wb are formed once and multiplied (tan = sin/cos is the only per-stage division, sec^2 = 1+tan^2).
 * Matrices here are dense and row-major; the kernel skips structural zeros/ones of A and B, which is
 * exact (x*1 = x, x + 0 = x, fmaf(0, y, z) = z for finite y).
 */
#define _GNU_SOURCE
#include <math.h>
#include <stdint.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "crb_oracle_mpc.h"

#include <stdio.h>
int crb_oracle_mpc_trace = 0; /* debugging aid: print one line per outer iteration to stderr */
int64_t crb_oracle_mpc_nfw_hist[64][16]; /* debugging aid: [outer iteration][forward sweeps used] */

/* ---- sin/cos: Cody-Waite reduction by pi/2 + Cephes-style minimax polynomials ------------------- */
void crb_oracle_sincosf(float x, float* sn, float* cs) {
  if (!(fabsf(x) <= 1.0e5f)) { /* also catches NaN */
    *sn = x - x;
    *cs = x - x;
    if (fabsf(x) > 1.0e5f && x - x == 0.0f) { /* finite but huge: no accuracy promised */
      *sn = 0.0f;
      *cs = 1.0f;
    }
    return;
  }
  const float j = rintf(x * 0.63661977236758134308f);
  float r = fmaf(-j, 1.5707962512969970703125f, x);
  r = fmaf(-j, 7.5497894158615963533521e-08f, r);
  r = fmaf(-j, 5.3903029534742383e-15f, r);
  const int q = (int)j & 3;
  const float z = r * r;
  float ps = fmaf(z, -1.9515295891e-4f, 8.3321608736e-3f);
  ps = fmaf(ps, z, -1.6666654611e-1f);
  ps = ps * z;
  ps = fmaf(ps, r, r); /* sin(r) */
  float pc = fmaf(z, 2.443315711809948e-5f, -1.388731625493765e-3f);
  pc = fmaf(pc, z, 4.166664568298827e-2f);
  pc = pc * z;
  pc = fmaf(pc, z, fmaf(-0.5f, z, 1.0f)); /* cos(r) */
  float s_ = (q & 1) ? pc : ps;
  float c_ = (q & 1) ? ps : pc;
  if (q & 2) s_ = -s_;
  if ((q + 1) & 2) c_ = -c_;
  *sn = s_;
  *cs = c_;
}

/* ---- bounds on a_t that keep v_{t+1} = v_t + a_t*dt inside [min_speed, max_speed] (:298-301) ---- */
static void a_bounds(float v, const crb_oracle_mpc_params* p, float* lo, float* hi, int* lo_sp,
                     int* hi_sp) {
  const float inv_dt = 1.0f / p->dt;
  const float lo_v = (p->min_speed - v) * inv_dt;
  const float hi_v = (p->max_speed - v) * inv_dt;
  const float am = p->max_accel;
  float l = lo_v < am ? lo_v : am;
  l = l > -am ? l : -am;
  float h = hi_v > -am ? hi_v : -am;
  h = h < am ? h : am;
  *lo = l;
  *hi = h;
  *lo_sp = lo_v > -am;
  *hi_sp = hi_v < am;
}

static inline float clampf(float u, float lo, float hi) { return u < lo ? lo : (u > hi ? hi : u); }

/* one step of :242-245 with the shared trig; u = (delta, a) */
static void dyn_step(const float x[4], float delta, float a, const crb_oracle_mpc_params* p,
                     float xn[4]) {
  float s, c, sd, cd;
  crb_oracle_sincosf(x[2], &s, &c);
  crb_oracle_sincosf(delta, &sd, &cd);
  const float kap = (sd / cd) * (1.0f / p->wb);
  const float vdt = x[3] * p->dt;
  xn[0] = fmaf(vdt, c, x[0]);
  xn[1] = fmaf(vdt, s, x[1]);
  xn[2] = fmaf(vdt, kap, x[2]);
  xn[3] = fmaf(a, p->dt, x[3]);
}

/* fg[0] (:199-250) evaluated directly on a roll-out: X[t][4], U[t][2] = (delta, a), xref[t][4] */
static float direct_cost(int T, const float X[][4], const float U[][2], const float xref[][4],
                         const crb_oracle_mpc_params* p) {
  const float wq[4] = {p->w_x, p->w_y, p->w_yaw, p->w_v};
  float J = 0.0f;
  for (int t = 0; t < T - 1; ++t) {
    J = fmaf(p->w_delta * U[t][0], U[t][0], J);
    J = fmaf(p->w_a * U[t][1], U[t][1], J);
    if (t >= 1) {
      const float dd = U[t][0] - U[t - 1][0];
      const float da = U[t][1] - U[t - 1][1];
      J = fmaf(p->w_ddelta * dd, dd, J);
      J = fmaf(p->w_da * da, da, J);
    }
    for (int k = 0; k < 4; ++k) {
      const float e = X[t + 1][k] - xref[t + 1][k];
      J = fmaf(wq[k] * e, e, J);
    }
  }
  return J;
}

/* ---- dense helpers (row-major, ascending-index fmaf chains) --------------------------------------- */
/* C[r x c] = A[r x k] * B[k x c] */
static void mm(const float* A, const float* B, float* C, int r, int k, int c) {
  for (int i = 0; i < r; ++i)
    for (int j = 0; j < c; ++j) {
      float acc = A[i * k + 0] * B[0 * c + j];
      for (int l = 1; l < k; ++l) acc = fmaf(A[i * k + l], B[l * c + j], acc);
      C[i * c + j] = acc;
    }
}
/* C[r x c] = A^T * B with A [k x r], B [k x c] */
static void mtm(const float* A, const float* B, float* C, int r, int k, int c) {
  for (int i = 0; i < r; ++i)
    for (int j = 0; j < c; ++j) {
      float acc = A[0 * r + i] * B[0 * c + j];
      for (int l = 1; l < k; ++l) acc = fmaf(A[l * r + i], B[l * c + j], acc);
      C[i * c + j] = acc;
    }
}

typedef struct {
  float k[2];
  float Kx[2][4];
  float Kw[2][2];
} stage_gain;

#define REG_EPS 1.0e-3f

typedef struct {
  float k[2];      /* minimiser (du) */
  int cl[2];       /* clamped flags */
  float H00, H11;  /* regularised diagonal used for the gains (H01 is never changed) */
  float idet, ih00, ih11;
} qp_result;

/* Projected-Newton step for min 0.5 u'Qu + g'u over the box [lo, hi]^2 (which contains 0); Q may be
 * indefinite.  1. Inputs that sit on a bound with the gradient pushing outward are fixed first
 * (Bertsekas' strongly active set).  2. The Hessian of the remaining inputs is made positive definite
 * using the curvature MAGNITUDE (1-D: max(|Qjj|, eps); 2-D: shift so that the smallest eigenvalue
 * becomes max(|lam_min|, eps)), so that a noise-level gradient gives a noise-level step.  3. The convex box QP in those inputs is solved exactly:
 * interior point if feasible, else the best of the four clamped edge minimisers (edge order u0 = lo0,
 * hi0, u1 = lo1, hi1; strict '<' keeps the first). */
static void box_qp2(float Q00, float Q01, float Q11, const float g[2], const float lo[2],
                    const float hi[2], qp_result* r) {
  const int sa0lo = lo[0] >= 0.0f && g[0] > 0.0f, sa0hi = !sa0lo && hi[0] <= 0.0f && g[0] < 0.0f;
  const int sa1lo = lo[1] >= 0.0f && g[1] > 0.0f, sa1hi = !sa1lo && hi[1] <= 0.0f && g[1] < 0.0f;
  const int sa0 = sa0lo || sa0hi, sa1 = sa1lo || sa1hi;
  r->H00 = Q00; r->H11 = Q11; r->idet = 0.0f; r->ih00 = 0.0f; r->ih11 = 0.0f;
  r->k[0] = 0.0f; r->k[1] = 0.0f;
  if (sa0) r->k[0] = sa0lo ? lo[0] : hi[0];
  if (sa1) r->k[1] = sa1lo ? lo[1] : hi[1];
  if (sa0 && sa1) { r->cl[0] = 1; r->cl[1] = 1; return; }
  if (sa0) { /* u1 free, 1-D */
    r->H11 = fabsf(Q11) > REG_EPS ? fabsf(Q11) : REG_EPS; /* curvature magnitude */
    r->ih11 = 1.0f / r->H11;
    float uj = -(fmaf(Q01, r->k[0], g[1]) * r->ih11);
    int cj = 0;
    if (uj <= lo[1]) { uj = lo[1]; cj = 1; }
    else if (uj >= hi[1]) { uj = hi[1]; cj = 1; }
    r->k[1] = uj; r->cl[0] = 1; r->cl[1] = cj;
    return;
  }
  if (sa1) { /* u0 free, 1-D */
    r->H00 = fabsf(Q00) > REG_EPS ? fabsf(Q00) : REG_EPS;
    r->ih00 = 1.0f / r->H00;
    float uj = -(fmaf(Q01, r->k[1], g[0]) * r->ih00);
    int cj = 0;
    if (uj <= lo[0]) { uj = lo[0]; cj = 1; }
    else if (uj >= hi[0]) { uj = hi[0]; cj = 1; }
    r->k[0] = uj; r->cl[1] = 1; r->cl[0] = cj;
    return;
  }
  /* both free: shift to positive definite, then the convex 2-D box QP */
  const float mh = 0.5f * (Q00 + Q11), dh = 0.5f * (Q00 - Q11);
  const float lam = mh - sqrtf(fmaf(dh, dh, Q01 * Q01));
  /* smallest eigenvalue -> max(|lam|, eps): steps scale with the curvature magnitude */
  const float shift = lam < REG_EPS ? (-lam > REG_EPS ? -lam : REG_EPS) - lam : 0.0f;
  const float H00 = Q00 + shift, H11 = Q11 + shift, H01 = Q01;
  const float det = fmaf(H00, H11, -(H01 * H01));
  const float idet = 1.0f / det, ih00 = 1.0f / H00, ih11 = 1.0f / H11;
  r->H00 = H00; r->H11 = H11; r->idet = idet; r->ih00 = ih00; r->ih11 = ih11;
  const float n0 = fmaf(H01, g[1], -(H11 * g[0]));
  const float n1 = fmaf(H01, g[0], -(H00 * g[1]));
  const float u0 = n0 * idet, u1 = n1 * idet;
  if (u0 >= lo[0] && u0 <= hi[0] && u1 >= lo[1] && u1 <= hi[1]) {
    r->k[0] = u0; r->k[1] = u1; r->cl[0] = 0; r->cl[1] = 0;
    return;
  }
  const float Hd[2] = {H00, H11};
  const float ih[2] = {ih00, ih11};
  float best = INFINITY;
  r->k[0] = lo[0] > 0.0f ? lo[0] : (hi[0] < 0.0f ? hi[0] : 0.0f); /* only kept if every edge is NaN */
  r->k[1] = lo[1] > 0.0f ? lo[1] : (hi[1] < 0.0f ? hi[1] : 0.0f);
  r->cl[0] = 1; r->cl[1] = 1;
  for (int i = 0; i < 2; ++i) {
    const int j = 1 - i;
    for (int side = 0; side < 2; ++side) {
      const float b = side ? hi[i] : lo[i];
      float uj = -(fmaf(H01, b, g[j]) * ih[j]);
      int cj = 0;
      if (uj <= lo[j]) { uj = lo[j]; cj = 1; }
      else if (uj >= hi[j]) { uj = hi[j]; cj = 1; }
      const float ti = fmaf(0.5f * Hd[i], b, g[i]);
      const float tj = fmaf(0.5f * Hd[j], uj, g[j]);
      const float val = fmaf(ti, b, fmaf(tj, uj, (H01 * b) * uj));
      if (val < best) {
        best = val;
        r->k[i] = b; r->k[j] = uj; r->cl[i] = 1; r->cl[j] = cj;
      }
    }
  }
}

static void backward_sweep(int T, const float X[][4], const float U[][2], const float xref[][4],
                           const crb_oracle_mpc_params* p, int gn, stage_gain* gains) {
  const int N = T - 1;
  const float R2[2] = {2.0f * p->w_delta, 2.0f * p->w_a};
  const float Rd2[2] = {2.0f * p->w_ddelta, 2.0f * p->w_da};
  const float Q2[4] = {2.0f * p->w_x, 2.0f * p->w_y, 2.0f * p->w_yaw, 2.0f * p->w_v};
  const float dt = p->dt, inv_wb = 1.0f / p->wb, inv_dt = 1.0f / p->dt;
  float Pxx[16], Pxw[8], Pww[4], px[4], pw[2];
  memset(Pxx, 0, sizeof(Pxx)); memset(Pxw, 0, sizeof(Pxw)); memset(Pww, 0, sizeof(Pww));
  for (int i = 0; i < 4; ++i) {
    Pxx[i * 4 + i] = Q2[i];
    px[i] = Q2[i] * (X[N][i] - xref[N][i]);
  }
  pw[0] = pw[1] = 0.0f;

  for (int t = N - 1; t >= 0; --t) {
    const int hr = t >= 1;
    const float yaw = X[t][2], v = X[t][3], delta = U[t][0];
    float s, c, sd, cd;
    crb_oracle_sincosf(yaw, &s, &c);
    crb_oracle_sincosf(delta, &sd, &cd);
    const float tn = sd / cd;
    const float kap = tn * inv_wb;
    const float vdt = v * dt;
    const float bv = (dt * inv_wb) * fmaf(tn, tn, 1.0f); /* dt / (wb cos^2) with sec^2 = 1 + tan^2 */
    const float B20 = v * bv;
    float A[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    A[0 * 4 + 2] = -(vdt * s);
    A[0 * 4 + 3] = c * dt;
    A[1 * 4 + 2] = vdt * c;
    A[1 * 4 + 3] = s * dt;
    A[2 * 4 + 3] = kap * dt;
    float B[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    B[2 * 2 + 0] = B20;
    B[3 * 2 + 1] = dt;

    /* gradients */
    float qx[4], qu[2], qw[2], du[2] = {0.0f, 0.0f};
    mtm(A, px, qx, 4, 4, 1);
    if (hr)
      for (int i = 0; i < 4; ++i) qx[i] = fmaf(Q2[i], X[t][i] - xref[t][i], qx[i]);
    float BtPx[2];
    mtm(B, px, BtPx, 2, 4, 1);
    for (int i = 0; i < 2; ++i) {
      if (hr) du[i] = U[t][i] - U[t - 1][i];
      float g = R2[i] * U[t][i];
      if (hr) g = fmaf(Rd2[i], du[i], g);
      g = g + BtPx[i];
      g = g + pw[i];
      qu[i] = g;
      qw[i] = hr ? -(Rd2[i] * du[i]) : 0.0f;
    }
    /* second derivatives of the dynamics contracted with the costate px (p0,p1,p2) */
    /* (skipped in Gauss-Newton mode, gn) */
    const float hyy = gn ? 0.0f : -(vdt * fmaf(px[1], s, px[0] * c));
    const float hyv = gn ? 0.0f : dt * fmaf(px[1], c, -(px[0] * s));
    /* Hessian blocks */
    float G[16], Qxx[16];
    mm(Pxx, A, G, 4, 4, 4);
    mtm(A, G, Qxx, 4, 4, 4);
    if (hr)
      for (int i = 0; i < 4; ++i) Qxx[i * 4 + i] = Qxx[i * 4 + i] + Q2[i];
    Qxx[2 * 4 + 2] = Qxx[2 * 4 + 2] + hyy;
    Qxx[2 * 4 + 3] = Qxx[2 * 4 + 3] + hyv;
    Qxx[3 * 4 + 2] = Qxx[3 * 4 + 2] + hyv;
    float Pwx[8], W[8], BtG[8], Qux[8];
    for (int i = 0; i < 4; ++i)
      for (int a = 0; a < 2; ++a) Pwx[a * 4 + i] = Pxw[i * 2 + a];
    mm(Pwx, A, W, 2, 4, 4);
    mtm(B, G, BtG, 2, 4, 4);
    for (int i = 0; i < 8; ++i) Qux[i] = BtG[i] + W[i];
    if (!gn) Qux[0 * 4 + 3] = fmaf(px[2], bv, Qux[0 * 4 + 3]);
    float PB[8], BtPB[4], BtPxw[4];
    mm(Pxx, B, PB, 4, 4, 2);
    mtm(B, PB, BtPB, 2, 4, 2);
    mtm(B, Pxw, BtPxw, 2, 4, 2);
    const float L0 = hr ? R2[0] + Rd2[0] : R2[0];
    const float L1 = hr ? R2[1] + Rd2[1] : R2[1];
    float Q00 = (((L0 + BtPB[0]) + BtPxw[0]) + BtPxw[0]) + Pww[0];
    float Q01 = (((0.0f + BtPB[1]) + BtPxw[1]) + BtPxw[2]) + Pww[1];
    float Q11 = (((L1 + BtPB[3]) + BtPxw[3]) + BtPxw[3]) + Pww[3];
    if (!gn) Q00 = fmaf(px[2], (2.0f * tn) * B20, Q00);
    const float Quw[2] = {hr ? -Rd2[0] : 0.0f, hr ? -Rd2[1] : 0.0f}; /* diagonal */
    const float Qww[2] = {hr ? Rd2[0] : 0.0f, hr ? Rd2[1] : 0.0f};   /* diagonal */

    /* box on du = u - ubar */
    float alo, ahi;
    int lo_sp, hi_sp;
    a_bounds(v, p, &alo, &ahi, &lo_sp, &hi_sp);
    const float lo[2] = {-p->max_steer - U[t][0], alo - U[t][1]};
    const float hi[2] = {p->max_steer - U[t][0], ahi - U[t][1]};
    stage_gain* gn_ = &gains[t];
    /* Quu may be indefinite (exact second derivatives): projected-Newton box QP; the gains use the
     * regularised Hessian of the free inputs, the value update below uses the true Quu */
    qp_result qp;
    box_qp2(Q00, Q01, Q11, qu, lo, hi, &qp);
    const int cl[2] = {qp.cl[0], qp.cl[1]};
    gn_->k[0] = qp.k[0]; gn_->k[1] = qp.k[1];
    const float H00 = qp.H00, H11 = qp.H11, H01 = Q01;
    const float idet = qp.idet, ih00 = qp.ih00, ih11 = qp.ih11;
    memset(gn_->Kx, 0, sizeof(gn_->Kx));
    memset(gn_->Kw, 0, sizeof(gn_->Kw));
    if (cl[1]) { /* a speed-induced bound on a moves with v: da/dv = -1/dt */
      const int at_lo = gn_->k[1] <= lo[1];
      if ((at_lo && lo_sp) || (!at_lo && hi_sp)) gn_->Kx[1][3] = -inv_dt;
    }
    if (!cl[0] && !cl[1]) {
      for (int j = 0; j < 4; ++j) {
        gn_->Kx[0][j] = fmaf(H01, Qux[1 * 4 + j], -(H11 * Qux[0 * 4 + j])) * idet;
        gn_->Kx[1][j] = fmaf(H01, Qux[0 * 4 + j], -(H00 * Qux[1 * 4 + j])) * idet;
      }
      /* Quw is diagonal: column 0 = (Quw0, 0), column 1 = (0, Quw1) */
      gn_->Kw[0][0] = fmaf(H01, 0.0f, -(H11 * Quw[0])) * idet;
      gn_->Kw[1][0] = fmaf(H01, Quw[0], -(H00 * 0.0f)) * idet;
      gn_->Kw[0][1] = fmaf(H01, Quw[1], -(H11 * 0.0f)) * idet;
      gn_->Kw[1][1] = fmaf(H01, 0.0f, -(H00 * Quw[1])) * idet;
    } else if (!cl[0] || !cl[1]) {
      const int j = cl[0] ? 1 : 0, i = 1 - j;
      const float ihjj = j ? ih11 : ih00;
      for (int col = 0; col < 4; ++col)
        gn_->Kx[j][col] = -(fmaf(H01, gn_->Kx[i][col], Qux[j * 4 + col]) * ihjj);
      for (int col = 0; col < 2; ++col) {
        const float quw_jc = (col == j) ? Quw[j] : 0.0f;
        gn_->Kw[j][col] = -(fmaf(H01, gn_->Kw[i][col], quw_jc) * ihjj);
      }
    }
    /* value-function update for the affine policy du = k + Kx dx + Kw dw, with the TRUE Quu */
    const float k0 = gn_->k[0], k1 = gn_->k[1];
    const float m0 = fmaf(Q01, k1, fmaf(Q00, k0, qu[0]));
    const float m1 = fmaf(Q11, k1, fmaf(Q01, k0, qu[1]));
    float Mx[2][4], Mw[2][2];
    for (int j = 0; j < 4; ++j) {
      Mx[0][j] = fmaf(Q01, gn_->Kx[1][j], fmaf(Q00, gn_->Kx[0][j], Qux[0 * 4 + j]));
      Mx[1][j] = fmaf(Q11, gn_->Kx[1][j], fmaf(Q01, gn_->Kx[0][j], Qux[1 * 4 + j]));
    }
    for (int b = 0; b < 2; ++b) {
      Mw[0][b] = fmaf(Q01, gn_->Kw[1][b], fmaf(Q00, gn_->Kw[0][b], b == 0 ? Quw[0] : 0.0f));
      Mw[1][b] = fmaf(Q11, gn_->Kw[1][b], fmaf(Q01, gn_->Kw[0][b], b == 1 ? Quw[1] : 0.0f));
    }
    float npx[4], npw[2], nPxx[16], nPxw[8], nPww[4];
    for (int i = 0; i < 4; ++i) {
      float acc = qx[i];
      acc = fmaf(gn_->Kx[0][i], m0, acc);
      acc = fmaf(gn_->Kx[1][i], m1, acc);
      acc = fmaf(Qux[0 * 4 + i], k0, acc);
      acc = fmaf(Qux[1 * 4 + i], k1, acc);
      npx[i] = acc;
    }
    for (int b = 0; b < 2; ++b) {
      float acc = qw[b];
      acc = fmaf(gn_->Kw[0][b], m0, acc);
      acc = fmaf(gn_->Kw[1][b], m1, acc);
      acc = fmaf(Quw[b], b == 0 ? k0 : k1, acc);
      npw[b] = acc;
    }
    for (int i = 0; i < 4; ++i)
      for (int j = 0; j <= i; ++j) {
        float acc = Qxx[i * 4 + j];
        acc = fmaf(gn_->Kx[0][i], Mx[0][j], acc);
        acc = fmaf(gn_->Kx[1][i], Mx[1][j], acc);
        acc = fmaf(Qux[0 * 4 + i], gn_->Kx[0][j], acc);
        acc = fmaf(Qux[1 * 4 + i], gn_->Kx[1][j], acc);
        nPxx[i * 4 + j] = acc;
        nPxx[j * 4 + i] = acc;
      }
    for (int i = 0; i < 4; ++i)
      for (int b = 0; b < 2; ++b) {
        float acc = gn_->Kx[0][i] * Mw[0][b];
        acc = fmaf(gn_->Kx[1][i], Mw[1][b], acc);
        acc = fmaf(Qux[0 * 4 + i], gn_->Kw[0][b], acc);
        acc = fmaf(Qux[1 * 4 + i], gn_->Kw[1][b], acc);
        nPxw[i * 2 + b] = acc;
      }
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b <= a; ++b) {
        float acc = a == b ? Qww[a] : 0.0f;
        acc = fmaf(gn_->Kw[0][a], Mw[0][b], acc);
        acc = fmaf(gn_->Kw[1][a], Mw[1][b], acc);
        acc = fmaf(Quw[a], gn_->Kw[a][b], acc); /* sum_c Quw[c][a] Kw[c][b], Quw diagonal */
        nPww[a * 2 + b] = acc;
        nPww[b * 2 + a] = acc;
      }
    memcpy(Pxx, nPxx, sizeof(Pxx)); memcpy(Pxw, nPxw, sizeof(Pxw)); memcpy(Pww, nPww, sizeof(Pww));
    memcpy(px, npx, sizeof(px)); memcpy(pw, npw, sizeof(pw));
  }
}

/* clamped roll-out under the affine policy; returns dJ (accurate cost difference) and du */
static void forward_sweep(int T, const float x0[4], const float X[][4], const float U[][2],
                          const float xref[][4], const stage_gain* gains, float alpha,
                          const crb_oracle_mpc_params* p, float Xn[][4], float Un[][2], float* dJ_out,
                          float* du_out) {
  const float wq[4] = {p->w_x, p->w_y, p->w_yaw, p->w_v};
  float dJ = 0.0f, dus = 0.0f;
  for (int i = 0; i < 4; ++i) Xn[0][i] = x0[i];
  for (int t = 0; t < T - 1; ++t) {
    const stage_gain* g = &gains[t];
    float dx[4], dw[2] = {0.0f, 0.0f};
    for (int i = 0; i < 4; ++i) dx[i] = Xn[t][i] - X[t][i];
    if (t >= 1)
      for (int i = 0; i < 2; ++i) dw[i] = Un[t - 1][i] - U[t - 1][i];
    float u[2];
    for (int i = 0; i < 2; ++i) {
      float acc = fmaf(alpha, g->k[i], U[t][i]);
      for (int j = 0; j < 4; ++j) acc = fmaf(g->Kx[i][j], dx[j], acc);
      for (int j = 0; j < 2; ++j) acc = fmaf(g->Kw[i][j], dw[j], acc);
      u[i] = acc;
    }
    u[0] = clampf(u[0], -p->max_steer, p->max_steer);
    float alo, ahi;
    int s0, s1;
    a_bounds(Xn[t][3], p, &alo, &ahi, &s0, &s1);
    u[1] = clampf(u[1], alo, ahi);
    Un[t][0] = u[0];
    Un[t][1] = u[1];
    dyn_step(Xn[t], u[0], u[1], p, Xn[t + 1]);
    /* cost difference, term by term */
    const float wu[2] = {p->w_delta, p->w_a};
    const float wd[2] = {p->w_ddelta, p->w_da};
    for (int i = 0; i < 2; ++i) {
      const float d = u[i] - U[t][i], s = u[i] + U[t][i];
      dJ = fmaf(wu[i] * d, s, dJ);
      dus = dus + fabsf(d);
    }
    if (t >= 1)
      for (int i = 0; i < 2; ++i) {
        const float qn = u[i] - Un[t - 1][i], qo = U[t][i] - U[t - 1][i];
        dJ = fmaf(wd[i] * (qn - qo), qn + qo, dJ);
      }
    for (int k = 0; k < 4; ++k) {
      const float en = Xn[t + 1][k] - xref[t + 1][k], eo = X[t + 1][k] - xref[t + 1][k];
      dJ = fmaf(wq[k] * (Xn[t + 1][k] - X[t + 1][k]), en + eo, dJ);
    }
  }
  *dJ_out = dJ;
  *du_out = dus;
}

void crb_oracle_mpc_solve(int T, const float x0_in[4], const float* xref_flat /*[T][4]*/,
                          const float* u_init /*[T-1][2] (delta,a) or NULL*/,
                          const crb_oracle_mpc_params* p, float* sol /*[4T+2(T-1)] ref layout or NULL*/,
                          float u0_out[2] /*(a0, delta0)*/, float* cost_out, int32_t* status_out,
                          int32_t* iters_out) {
  float XA[CRB_ORACLE_MPC_MAX_T][4], XB[CRB_ORACLE_MPC_MAX_T][4];
  float UA[CRB_ORACLE_MPC_MAX_T][2], UB[CRB_ORACLE_MPC_MAX_T][2];
  float xref[CRB_ORACLE_MPC_MAX_T][4];
  stage_gain gains[CRB_ORACLE_MPC_MAX_T];
  float(*X)[4] = XA, (*Xn)[4] = XB;
  float(*U)[2] = UA, (*Un)[2] = UB;
  const int N = T - 1;
  /* Work in the frame translated to the initial position: cost and dynamics only see x - xref and
   * are translation invariant, and binary32 keeps ~16x more absolute resolution at |x| ~ 20 m than at
   * the course coordinates (~400 m).  The offset is added back on output. */
  const float ox = x0_in[0], oy = x0_in[1];
  const float x0[4] = {0.0f, 0.0f, x0_in[2], x0_in[3]};
  for (int t = 0; t < T; ++t) {
    xref[t][0] = xref_flat[t * 4 + 0] - ox;
    xref[t][1] = xref_flat[t * 4 + 1] - oy;
    xref[t][2] = xref_flat[t * 4 + 2];
    xref[t][3] = xref_flat[t * 4 + 3];
  }
  /* initial clamped roll-out (cold start: zeros, :266-269) */
  for (int i = 0; i < 4; ++i) X[0][i] = x0[i];
  for (int t = 0; t < N; ++t) {
    float d = u_init ? u_init[t * 2 + 0] : 0.0f;
    float a = u_init ? u_init[t * 2 + 1] : 0.0f;
    d = clampf(d, -p->max_steer, p->max_steer);
    float alo, ahi;
    int s0, s1;
    a_bounds(X[t][3], p, &alo, &ahi, &s0, &s1);
    a = clampf(a, alo, ahi);
    U[t][0] = d;
    U[t][1] = a;
    dyn_step(X[t], d, a, p, X[t + 1]);
  }
  int status = CRB_ORACLE_MPC_MAX_ITER, iters = 0;
  float J0 = direct_cost(T, (const float(*)[4])X, (const float(*)[2])U, (const float(*)[4])xref, p);
  if (!(fabsf(J0) <= 3.0e38f)) {
    status = CRB_ORACLE_MPC_NONFINITE;
  } else {
    int gn = 0; /* 0: Newton (exact second derivatives); 1: Gauss-Newton retry after a failed search */
    float Jc = J0; /* running cost: J0 plus the accepted differences */
    while (iters < p->max_iter) {
      backward_sweep(T, (const float(*)[4])X, (const float(*)[2])U, (const float(*)[4])xref, p, gn,
                     gains);
      ++iters;
      int accepted = 0, tiny = 0, jacc = 0;
      float dJ = 0.0f, du = 0.0f, alpha = 1.0f;
      for (int j = 0; j <= p->max_ls; ++j) {
        forward_sweep(T, x0, (const float(*)[4])X, (const float(*)[2])U, (const float(*)[4])xref,
                      gains, alpha, p, Xn, Un, &dJ, &du);
        /* the FULL step moves the inputs by <= du_th, or the cost by less than binary32 can resolve */
        if (j == 0) tiny = (du <= p->du_th) || (fabsf(dJ) <= p->j_tol * fabsf(Jc));
        if (dJ < 0.0f) { accepted = 1; jacc = j; break; }
        if (tiny) break;
        alpha = alpha * 0.5f;
      }
      if (crb_oracle_mpc_trace == 2) {
        int nf = 0; float a2 = 1.0f; while (a2 > alpha && nf < 14) { a2 *= 0.5f; ++nf; }
        nf = accepted || tiny ? nf + 1 : nf;
#pragma omp atomic
        crb_oracle_mpc_nfw_hist[iters < 64 ? iters - 1 : 63][nf < 16 ? nf : 15]++;
      }
      if (crb_oracle_mpc_trace == 1)
        fprintf(stderr, "  it %d gn %d accepted %d tiny %d alpha %g dJ %.3e du %.3e J %.6f\n", iters, gn,
                accepted, tiny, (double)alpha, (double)dJ, (double)du, (double)Jc);
      if (!accepted) {
        if (tiny) { status = CRB_ORACLE_MPC_CONVERGED; break; }
        if (!gn) { gn = 1; continue; }
        status = CRB_ORACLE_MPC_NO_DESCENT;
        break;
      }
      gn = 0;
      float(*tx)[4] = X; X = Xn; Xn = tx;
      float(*tu)[2] = U; U = Un; Un = tu;
      Jc = Jc + dJ;
      if ((jacc == 0 && tiny) || du <= p->du_th) { status = CRB_ORACLE_MPC_CONVERGED; break; }
    }
  }
  const float J = direct_cost(T, (const float(*)[4])X, (const float(*)[2])U, (const float(*)[4])xref, p);
  if (!(fabsf(J) <= 3.0e38f)) status = CRB_ORACLE_MPC_NONFINITE;
  if (sol) { /* reference layout :54-60 */
    for (int t = 0; t < T; ++t) {
      sol[0 * T + t] = X[t][0] + ox;
      sol[1 * T + t] = X[t][1] + oy;
      sol[2 * T + t] = X[t][2];
      sol[3 * T + t] = X[t][3];
    }
    for (int t = 0; t < N; ++t) {
      sol[4 * T + t] = U[t][0];
      sol[4 * T + N + t] = U[t][1];
    }
  }
  if (u0_out) { u0_out[0] = U[0][1]; u0_out[1] = U[0][0]; }
  if (cost_out) *cost_out = J;
  if (status_out) *status_out = status;
  if (iters_out) *iters_out = iters;
}

/* SoA batch with the libcrb layout: x0 [4][n], xref [4T][n] (field 4t+k), u_init [2(T-1)][n]
 * (delta block then a block), sol [4T+2(T-1)][n], u0 [2][n], cost/status/iters [n] */
void crb_oracle_mpc_solve_batched(int64_t n, int T, const float* x0, const float* xref,
                                  const float* u_init, const crb_oracle_mpc_params* p, float* sol,
                                  float* u0, float* cost, int32_t* status, int32_t* iters,
                                  int nthreads) {
  const int N = T - 1, nsol = 4 * T + 2 * N;
#ifdef _OPENMP
  if (nthreads <= 0) nthreads = omp_get_max_threads();
#pragma omp parallel for num_threads(nthreads) schedule(dynamic, 64)
#endif
  for (int64_t i = 0; i < n; ++i) {
    float x[4], xr[CRB_ORACLE_MPC_MAX_T * 4], ui[CRB_ORACLE_MPC_MAX_T * 2];
    float so[6 * CRB_ORACLE_MPC_MAX_T], u0o[2], c;
    int32_t st, itn;
    for (int k = 0; k < 4; ++k) x[k] = x0[k * n + i];
    for (int f = 0; f < 4 * T; ++f) xr[f] = xref[(int64_t)f * n + i];
    if (u_init)
      for (int t = 0; t < N; ++t) {
        ui[t * 2 + 0] = u_init[(int64_t)t * n + i];
        ui[t * 2 + 1] = u_init[(int64_t)(N + t) * n + i];
      }
    crb_oracle_mpc_solve(T, x, xr, u_init ? ui : 0, p, so, u0o, &c, &st, &itn);
    if (sol)
      for (int f = 0; f < nsol; ++f) sol[(int64_t)f * n + i] = so[f];
    if (u0) { u0[i] = u0o[0]; u0[n + i] = u0o[1]; }
    if (cost) cost[i] = c;
    if (status) status[i] = st;
    if (iters) iters[i] = itn;
  }
}

/* ---- update(): src/model_predictive_control.cpp:69-81 (plant step on the first control).
 * MAX_STEER, DT, WB, MAX_SPEED, MIN_SPEED are double macros: float operands promote to double and the
 * result narrows on assignment; std::cos/std::sin of a float are the float overloads; CppAD::tan of a
 * float resolves to std::tan(float).  k = {MAX_STEER, DT, WB, MAX_SPEED, MIN_SPEED}: the macros' values, or any
 * other constants in double (libcrb's promotion rule, crb.h, is applied by the caller). */
void crb_oracle_plant_update_k(float st[4], float a, float delta, const double k[5]) {
  const double MAX_STEER = k[0], DT = k[1], WB = k[2];
  const double MAX_SPEED = k[3], MIN_SPEED = k[4];
  if ((double)delta >= MAX_STEER) delta = (float)MAX_STEER;
  if ((double)delta <= -MAX_STEER) delta = (float)(-MAX_STEER);
  const float x = st[0], y = st[1], yaw = st[2], v = st[3];
  st[0] = (float)((double)x + (double)(v * cosf(yaw)) * DT);
  st[1] = (float)((double)y + (double)(v * sinf(yaw)) * DT);
  st[2] = (float)((double)yaw + (double)v / WB * (double)tanf(delta) * DT);
  st[3] = (float)((double)v + (double)a * DT);
  if ((double)st[3] > MAX_SPEED) st[3] = (float)MAX_SPEED;
  if ((double)st[3] < MIN_SPEED) st[3] = (float)MIN_SPEED;
}

void crb_oracle_plant_update(float st[4], float a, float delta) {
  const double k[5] = {45.0 / 180 * M_PI, 0.2, 2.5, 55.0 / 3.6, -20.0 / 3.6};
  crb_oracle_plant_update_k(st, a, delta, k);
}

/* ---- calc_nearest_index :107-127.  `ind` is a float in the reference (:109); the window is
 * [pind, pind+N_IND_SEARCH) with no bounds check (:110) — clipped to the course here. */
int crb_oracle_calc_nearest_index(const float st[4], const float* cx, const float* cy, int ncourse,
                                  int pind) {
  float mind = 3.402823466e+38f; /* std::numeric_limits<float>::max() */
  float ind = 0;
  for (unsigned int i = (unsigned int)pind; i < (unsigned int)pind + 10u; ++i) {
    if ((int)i >= ncourse) break;
    const float idx = cx[i] - st[0];
    const float idy = cy[i] - st[1];
    const float d_e = idx * idx + idy * idy;
    if (d_e < mind) {
      mind = d_e;
      ind = (float)i;
    }
  }
  return (int)ind;
}

/* ---- calc_ref_trajectory :130-170; xref out as [T][4].  DT: the macro's 0.2, or any other step in double ---- */
void crb_oracle_calc_ref_trajectory_dt(const float st[4], const float* cx, const float* cy,
                                       const float* cyaw, const float* sp, int ncourse, float dl, int T,
                                       int* target_ind, float* xref /*[T][4]*/, double DT) {
  for (int i = 0; i < 4 * T; ++i) xref[i] = 0.0f;                                  /* :133 */
  int ind = crb_oracle_calc_nearest_index(st, cx, cy, ncourse, *target_ind);       /* :138 */
  if (*target_ind >= ind) ind = *target_ind;                                       /* :139 */
  xref[0] = cx[ind]; xref[1] = cy[ind]; xref[2] = cyaw[ind]; xref[3] = sp[ind];    /* :141-144 */
  float travel = 0.0f;
  for (int i = 0; i < T; ++i) {
    travel = (float)((double)travel + (double)fabsf(st[3]) * DT);                  /* :149 */
    const int dind = (int)roundf(travel / dl);                                     /* :150 */
    const int j = (ind + dind) < ncourse ? ind + dind : ncourse - 1;               /* :154-165 */
    xref[i * 4 + 0] = cx[j];
    xref[i * 4 + 1] = cy[j];
    xref[i * 4 + 2] = cyaw[j];
    xref[i * 4 + 3] = sp[j];
  }
  *target_ind = ind;                                                               /* :169 */
}

void crb_oracle_calc_ref_trajectory(const float st[4], const float* cx, const float* cy,
                                    const float* cyaw, const float* sp, int ncourse, float dl, int T,
                                    int* target_ind, float* xref /*[T][4]*/) {
  crb_oracle_calc_ref_trajectory_dt(st, cx, cy, cyaw, sp, ncourse, dl, T, target_ind, xref, 0.2);
}
