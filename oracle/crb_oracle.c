/* crb_oracle.c — CPU restatement of the EKF and particle-filter hot paths of onlytailei/CppRobotics.
 * TEST INFRASTRUCTURE ONLY (see crb_oracle.h for who may load it and for the parity-pinning note).
 *
 * Every function restates the cited reference lines with dense, textbook loops: the matrices are
 * built in full (including their structural zeros and ones) and multiplied entry by entry in plain
 * IEEE binary32 with separate multiply and add (build with -ffp-contract=off, no -mfma), which is
 * what Eigen's fixed-size lazy products compile to on the reference's default x86-64 target.
 * Column-major storage throughout, like Eigen: M(r,c) = M[r + rows*c].
 */
#include "crb_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

int crb_oracle_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

/* ---- tiny dense helpers ------------------------------------------------------------------------ */
/* C(ra x cb) = A(ra x ca) * B(ca x cb); inner sum order selectable for ca == 4 */
static void matmul(const float* A, int ra, int ca, const float* B, int cb, float* C, int order) {
  for (int j = 0; j < cb; ++j) {
    for (int i = 0; i < ra; ++i) {
      float s;
      if (order == CRB_ORDER_PAIRWISE && ca == 4) {
        float s01 = A[i + ra * 0] * B[0 + ca * j] + A[i + ra * 1] * B[1 + ca * j];
        float s23 = A[i + ra * 2] * B[2 + ca * j] + A[i + ra * 3] * B[3 + ca * j];
        s = s01 + s23;
      } else {
        s = A[i + ra * 0] * B[0 + ca * j];
        for (int k = 1; k < ca; ++k) s = s + A[i + ra * k] * B[k + ca * j];
      }
      C[i + ra * j] = s;
    }
  }
}
static void transpose(const float* A, int r, int c, float* At) {
  for (int i = 0; i < r; ++i)
    for (int j = 0; j < c; ++j) At[j + c * i] = A[i + r * j];
}

/* ---- motion_model: src/extended_kalman_filter.cpp:22-36 (same text at src/particle_filter.cpp:26-40)
 *   F_ = I4 (:24-27)   B_ = [DT*cos(yaw) 0; DT*sin(yaw) 0; 0 DT; 1 0] (:29-33)   return F_*x + B_*u (:35)
 * DT is a double literal, std::cos(float) returns float: entries are (float)(DT * (double)cosf()). */
void crb_oracle_motion_model(const float x[4], const float u[2], double dt, float out[4]) {
  float F[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  float B[8];
  B[0 + 4 * 0] = (float)(dt * (double)cosf(x[2]));
  B[1 + 4 * 0] = (float)(dt * (double)sinf(x[2]));
  B[2 + 4 * 0] = (float)0.0;
  B[3 + 4 * 0] = (float)1.0;
  B[0 + 4 * 1] = 0.0f;
  B[1 + 4 * 1] = 0.0f;
  B[2 + 4 * 1] = (float)dt;
  B[3 + 4 * 1] = (float)0.0;
  float Fx[4], Bu[4];
  matmul(F, 4, 4, x, 1, Fx, CRB_ORDER_SEQ);
  matmul(B, 4, 2, u, 1, Bu, CRB_ORDER_SEQ);
  for (int i = 0; i < 4; ++i) out[i] = Fx[i] + Bu[i];
}

/* ---- jacobF: src/extended_kalman_filter.cpp:38-47.  yaw = x(2), v = u(0) (:40-41);
 *   jF(0,2) = -DT*v*sin(yaw)  jF(0,3) = DT*cos(yaw)  jF(1,2) = DT*v*cos(yaw)  jF(1,3) = DT*sin(yaw)
 * evaluated left to right in double ((-DT*v)*sin) and narrowed on assignment. */
void crb_oracle_jacobF(const float x[4], const float u[2], double dt, float jF[16]) {
  for (int i = 0; i < 16; ++i) jF[i] = 0.0f;
  for (int i = 0; i < 4; ++i) jF[i + 4 * i] = 1.0f;
  float yaw = x[2];
  float v = u[0];
  jF[0 + 4 * 2] = (float)(-dt * (double)v * (double)sinf(yaw));
  jF[0 + 4 * 3] = (float)(dt * (double)cosf(yaw));
  jF[1 + 4 * 2] = (float)(dt * (double)v * (double)cosf(yaw));
  jF[1 + 4 * 3] = (float)(dt * (double)sinf(yaw));
}

/* ---- ekf_estimation: src/extended_kalman_filter.cpp:64-78 ---------------------------------------- */
void crb_oracle_ekf_estimation(float xEst[4], float PEst[16], const float z[2], const float u[2],
                               const float Q[16], const float R[4], double dt, int order) {
  float xPred[4], jF[16], jFt[16], T1[16], T2[16], PPred[16];
  crb_oracle_motion_model(xEst, u, dt, xPred);                 /* :67 */
  crb_oracle_jacobF(xPred, u, dt, jF);                         /* :68  (evaluated at xPred) */
  transpose(jF, 4, 4, jFt);
  matmul(jF, 4, 4, PEst, 4, T1, order);                        /* :69  (jF*PEst) */
  matmul(T1, 4, 4, jFt, 4, T2, order);                         /*      (...)*jF^T */
  for (int i = 0; i < 16; ++i) PPred[i] = T2[i] + Q[i];        /*      + Q */

  float jH[8] = {1, 0, 0, 1, 0, 0, 0, 0};                      /* :57-62, 2x4 col-major */
  float jHt[8];
  transpose(jH, 2, 4, jHt);
  float zPred[2];
  matmul(jH, 2, 4, xPred, 1, zPred, CRB_ORDER_SEQ);            /* :72 observation_model :50-55 */
  float y[2] = {z[0] - zPred[0], z[1] - zPred[1]};             /* :73 */
  float HP[8], S[4];
  matmul(jH, 2, 4, PPred, 4, HP, CRB_ORDER_SEQ);               /* :74 jH*PPred (selector: exact) */
  matmul(HP, 2, 4, jHt, 2, S, CRB_ORDER_SEQ);
  for (int i = 0; i < 4; ++i) S[i] = S[i] + R[i];
  /* S.inverse(): Eigen's size-2 closed form, one division then four products */
  float det = S[0] * S[3] - S[1] * S[2];
  float invdet = 1.0f / det;
  float Sinv[4];
  Sinv[0] = S[3] * invdet;
  Sinv[1] = -S[1] * invdet;
  Sinv[2] = -S[2] * invdet;
  Sinv[3] = S[0] * invdet;
  float PHt[8], K[8];
  matmul(PPred, 4, 4, jHt, 2, PHt, CRB_ORDER_SEQ);             /* :75 (PPred*jH^T) (selector: exact) */
  matmul(PHt, 4, 2, Sinv, 2, K, CRB_ORDER_SEQ);                /*     (...)*S^-1 */
  float Ky[4];
  matmul(K, 4, 2, y, 1, Ky, CRB_ORDER_SEQ);                    /* :76 */
  for (int i = 0; i < 4; ++i) xEst[i] = xPred[i] + Ky[i];
  float KH[16], M[16];
  matmul(K, 4, 2, jH, 4, KH, CRB_ORDER_SEQ);                   /* :77 K*jH */
  for (int j = 0; j < 4; ++j)
    for (int i = 0; i < 4; ++i) M[i + 4 * j] = (i == j ? 1.0f : 0.0f) - KH[i + 4 * j];
  matmul(M, 4, 4, PPred, 4, PEst, order);                      /* (I-K*jH)*PPred, not symmetrised */
}

void crb_oracle_ekf_estimation_f64(double xEst[4], double PEst[16], const double z[2],
                                   const double u[2], const double Q[16], const double R[4],
                                   double dt) {
  double xp[4], jF[16] = {0}, T1[16], PP[16];
  double c = cos(xEst[2]), s = sin(xEst[2]);
  xp[0] = xEst[0] + dt * c * u[0];
  xp[1] = xEst[1] + dt * s * u[0];
  xp[2] = xEst[2] + dt * u[1];
  xp[3] = xEst[3] + u[0];
  for (int i = 0; i < 4; ++i) jF[i + 4 * i] = 1.0;
  jF[0 + 4 * 2] = -dt * u[0] * sin(xp[2]);
  jF[0 + 4 * 3] = dt * cos(xp[2]);
  jF[1 + 4 * 2] = dt * u[0] * cos(xp[2]);
  jF[1 + 4 * 3] = dt * sin(xp[2]);
  for (int j = 0; j < 4; ++j)
    for (int i = 0; i < 4; ++i) {
      double a = 0;
      for (int k = 0; k < 4; ++k) a += jF[i + 4 * k] * PEst[k + 4 * j];
      T1[i + 4 * j] = a;
    }
  for (int j = 0; j < 4; ++j)
    for (int i = 0; i < 4; ++i) {
      double a = 0;
      for (int k = 0; k < 4; ++k) a += T1[i + 4 * k] * jF[j + 4 * k];
      PP[i + 4 * j] = a + Q[i + 4 * j];
    }
  double y0 = z[0] - xp[0], y1 = z[1] - xp[1];
  double S00 = PP[0] + R[0], S10 = PP[1] + R[1], S01 = PP[4] + R[2], S11 = PP[5] + R[3];
  double det = S00 * S11 - S10 * S01;
  double i00 = S11 / det, i10 = -S10 / det, i01 = -S01 / det, i11 = S00 / det;
  double K[8];
  for (int i = 0; i < 4; ++i) {
    K[i] = PP[i] * i00 + PP[i + 4] * i10;
    K[i + 4] = PP[i] * i01 + PP[i + 4] * i11;
  }
  for (int i = 0; i < 4; ++i) xEst[i] = xp[i] + K[i] * y0 + K[i + 4] * y1;
  for (int j = 0; j < 4; ++j)
    for (int i = 0; i < 4; ++i)
      PEst[i + 4 * j] = PP[i + 4 * j] - (K[i] * PP[0 + 4 * j] + K[i + 4] * PP[1 + 4 * j]);
}

void crb_oracle_ekf_step_batched(int64_t n, float* x, float* P, const float* z, const float* u,
                                 const float* Q, const float* R, double dt, int n_steps, int order,
                                 int nthreads) {
#ifdef _OPENMP
  if (nthreads <= 0) nthreads = omp_get_max_threads();
#pragma omp parallel for num_threads(nthreads) schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i) {
    float xe[4], Pe[16], zz[2], uu[2];
    for (int f = 0; f < 4; ++f) xe[f] = x[f * n + i];
    for (int f = 0; f < 16; ++f) Pe[f] = P[f * n + i];
    for (int s = 0; s < n_steps; ++s) {
      zz[0] = z[((int64_t)s * 2 + 0) * n + i];
      zz[1] = z[((int64_t)s * 2 + 1) * n + i];
      uu[0] = u[((int64_t)s * 2 + 0) * n + i];
      uu[1] = u[((int64_t)s * 2 + 1) * n + i];
      crb_oracle_ekf_estimation(xe, Pe, zz, uu, Q, R, dt, order);
    }
    for (int f = 0; f < 4; ++f) x[f * n + i] = xe[f];
    for (int f = 0; f < 16; ++f) P[f * n + i] = Pe[f];
  }
}

/* ---- gauss_likelihood: src/particle_filter.cpp:53-57
 *   float p = 1.0 / std::sqrt(2.0 * PI * sigma * sigma) * std::exp(-x * x / (2 * sigma * sigma));
 * prefactor in double, exponent and exp in float (std::exp(float) -> expf), product in double. */
float crb_oracle_gauss_likelihood(float x, float sigma, double pi) {
  double pre = 1.0 / sqrt(2.0 * pi * (double)sigma * (double)sigma);
  float e = expf(-x * x / (2 * sigma * sigma));
  float p = (float)(pre * (double)e);
  return p;
}

/* ---- one iteration of the particle loop: src/particle_filter.cpp:82-101 -------------------------- */
void crb_oracle_pf_particle(float x[4], float* w, const double g[2], const float u[2],
                            const float rsim_diag[2], const float* landmarks, int n_lm, float Q,
                            double dt, double pi) {
  float ud[2];
  ud[0] = (float)((double)u[0] + g[0] * (double)rsim_diag[0]);   /* :87 */
  ud[1] = (float)((double)u[1] + g[1] * (double)rsim_diag[1]);   /* :88 */
  float xn[4];
  crb_oracle_motion_model(x, ud, dt, xn);                          /* :90 */
  float ww = *w;
  for (int i = 0; i < n_lm; ++i) {                                 /* :92-99 */
    const float* item = landmarks + 3 * i;                         /* (range, lx, ly) */
    float dx = xn[0] - item[1];
    float dy = xn[1] - item[2];
    float prez = sqrtf(dx * dx + dy * dy);
    float dz = prez - item[0];
    ww = ww * crb_oracle_gauss_likelihood(dz, sqrtf(Q), pi);
  }
  for (int i = 0; i < 4; ++i) x[i] = xn[i];                        /* :100 */
  *w = ww;                                                         /* :101 */
}

/* ---- counter-based normals (no reference counterpart: the reference copies an mt19937 by value,
 * :78; the batched engine takes noise as an input array or draws it from Philox4x32-10) ---------- */
static inline void philox_round(uint32_t c[4], const uint32_t k[2]) {
  uint64_t p0 = (uint64_t)0xD2511F53u * c[0];
  uint64_t p1 = (uint64_t)0xCD9E8D57u * c[2];
  uint32_t n0 = (uint32_t)(p1 >> 32) ^ c[1] ^ k[0];
  uint32_t n1 = (uint32_t)p1;
  uint32_t n2 = (uint32_t)(p0 >> 32) ^ c[3] ^ k[1];
  uint32_t n3 = (uint32_t)p0;
  c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}
void crb_oracle_philox_normal2(uint64_t seed, uint64_t index, float g[2]) {
  uint32_t c[4] = {(uint32_t)index, (uint32_t)(index >> 32), 0u, 0u};
  uint32_t k[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
  for (int r = 0; r < 10; ++r) {
    philox_round(c, k);
    k[0] += 0x9E3779B9u;
    k[1] += 0xBB67AE85u;
  }
  float u1 = (float)(c[0] >> 9) * 1.1920928955078125e-07f + 5.9604644775390625e-08f; /* (0,1) */
  float u2 = (float)(c[1] >> 9) * 1.1920928955078125e-07f + 5.9604644775390625e-08f;
  float rad = sqrtf(-2.0f * logf(u1));
  float ang = 6.28318530717958647692f * u2;
  g[0] = rad * cosf(ang);
  g[1] = rad * sinf(ang);
}

void crb_oracle_pf_predict_weight_batched(int64_t n, float* px, float* pw, const float* noise,
                                          uint64_t seed, const float* landmarks, int n_lm,
                                          const float u[2], const float rsim_diag[2], float Q,
                                          double dt, double pi, int nthreads) {
#ifdef _OPENMP
  if (nthreads <= 0) nthreads = omp_get_max_threads();
#pragma omp parallel for num_threads(nthreads) schedule(static)
#endif
  for (int64_t i = 0; i < n; ++i) {
    float x[4], w = pw[i];
    double g[2];
    for (int f = 0; f < 4; ++f) x[f] = px[f * n + i];
    if (noise) {
      g[0] = (double)noise[i];
      g[1] = (double)noise[n + i];
    } else {
      float gf[2];
      crb_oracle_philox_normal2(seed, (uint64_t)i, gf);
      g[0] = (double)gf[0];
      g[1] = (double)gf[1];
    }
    crb_oracle_pf_particle(x, &w, g, u, rsim_diag, landmarks, n_lm, Q, dt, pi);
    for (int f = 0; f < 4; ++f) px[f * n + i] = x[f];
    pw[i] = w;
  }
}

/* ---- pf_localization tail: src/particle_filter.cpp:104-107 and calc_covariance :59-71.
 * The reference sums 100 floats in float; for 10^6 particles the batched engine accumulates in
 * double (documented deviation), so this restatement does too. */
void crb_oracle_pf_estimate(int64_t n, const float* px, float* pw, float xEst[4], float PEst[16],
                            double* sum_w) {
  double s = 0.0;
  for (int64_t i = 0; i < n; ++i) s += (double)pw[i];
  if (sum_w) *sum_w = s;
  float sf = (float)s;
  for (int64_t i = 0; i < n; ++i) pw[i] = pw[i] / sf;                 /* :104 */
  double m[4] = {0, 0, 0, 0};
  for (int64_t i = 0; i < n; ++i)
    for (int f = 0; f < 4; ++f) m[f] += (double)px[f * n + i] * (double)pw[i];   /* :106 */
  for (int f = 0; f < 4; ++f) xEst[f] = (float)m[f];
  double C[16] = {0};
  for (int64_t i = 0; i < n; ++i) {                                   /* :65-68 */
    double d[4];
    for (int f = 0; f < 4; ++f) d[f] = (double)(px[f * n + i] - xEst[f]);
    for (int c = 0; c < 4; ++c)
      for (int r = 0; r < 4; ++r) C[r + 4 * c] += (double)pw[i] * d[r] * d[c];
  }
  for (int k = 0; k < 16; ++k) PEst[k] = (float)C[k];
}

/* ---- verification aids for the arithmetic shortcuts the CUDA PF kernel takes -------------------------
 * (a) x / d for a launch-constant d computed without a divide: r = RN(1/d); q0 = x*r;
 *     rem = fma(-q0, d, x); q = fma(rem, r, q0).  Returns how many floats x with bit patterns in
 *     [lo_bits, hi_bits] give q != x / d (Markstein: none, barring under/overflow).
 * (b) (float)(pre * (double)e) computed in binary32 as a float-float product.  Returns the number of
 *     mismatches over the same range of e. */
int64_t crb_oracle_check_const_division(float d, uint32_t lo_bits, uint32_t hi_bits) {
  const float r = 1.0f / d;
  int64_t bad = 0;
#ifdef _OPENMP
#pragma omp parallel for reduction(+ : bad) schedule(static)
#endif
  for (int64_t b = (int64_t)lo_bits; b <= (int64_t)hi_bits; ++b) {
    uint32_t u = (uint32_t)b;
    float x;
    memcpy(&x, &u, 4);
    const float q0 = x * r;
    const float rem = fmaf(-q0, d, x);
    const float q = fmaf(rem, r, q0);
    const float ref = x / d;
    if (!(q == ref) && !(q != q && ref != ref)) ++bad;
  }
  return bad;
}
int64_t crb_oracle_check_ff_product(double pre, uint32_t lo_bits, uint32_t hi_bits) {
  const float ph_c = (float)pre;
  const float pl_c = (float)(pre - (double)ph_c);
  int64_t bad = 0;
#ifdef _OPENMP
#pragma omp parallel for reduction(+ : bad) schedule(static)
#endif
  for (int64_t b = (int64_t)lo_bits; b <= (int64_t)hi_bits; ++b) {
    uint32_t u = (uint32_t)b;
    float e;
    memcpy(&e, &u, 4);
    const float ph = ph_c * e;
    const float err = fmaf(ph_c, e, -ph);
    const float c = fmaf(pl_c, e, err);
    const float p = ph + c;
    const float ref = (float)(pre * (double)e);
    if (!(p == ref)) ++bad;
  }
  return bad;
}

/* (c) resampleid = (float)((double)(float)(j / NP) + U / NP) (:131-133) as crb_pf_gather2_kernel computes it
 *     (pf_resample_id_rcp): both quotients as q = a r, q += fma(-q, NP, a) r with r = RN(1 / NP).  Counts the
 *     (j, NP, U) where either double quotient is not the correctly rounded one or the float result differs:
 *     - every NP in [1, n_max] at j in {0, 1, 2, NP/2, NP-2, NP-1} and 32 hashed j;
 *     - every j in [0, NP) for each NP of ns[0..n_ns);
 *     - all 2^23 floats U in [1, 2) (the Philox draws) for each NP of ns, at a hashed j.
 *     Away from those j the U of a case is hashed too.  *evaluated receives the number of cases. */
static inline uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
static inline float u12_from_bits(uint32_t m) { return 1.0f + (float)(m & 0x7FFFFFu) * 1.1920928955078125e-07f; }
static inline int resample_id_rcp_bad(int64_t j, int64_t n, float U) {
  const double n_d = (double)n, inv_n = 1.0 / n_d;
  const double jd = (double)j;
  double q = jd * inv_n;
  q = fma(fma(-q, n_d, jd), inv_n, q);
  const double ud = (double)U;
  double t = ud * inv_n;
  t = fma(fma(-t, n_d, ud), inv_n, t);
  const float got = (float)((double)(float)q + t);
  const double q_ref = jd / n_d, t_ref = ud / n_d;
  const float want = (float)((double)(float)q_ref + t_ref);
  return q != q_ref || t != t_ref || got != want;
}
int64_t crb_oracle_check_resample_id_rcp(int64_t n_max, const int64_t* ns, int n_ns, int64_t* evaluated) {
  int64_t bad = 0, cnt = 0;
#ifdef _OPENMP
#pragma omp parallel for reduction(+ : bad, cnt) schedule(dynamic, 4096)
#endif
  for (int64_t n = 1; n <= n_max; ++n) {
    const int64_t fixed[6] = {0, 1, 2, n / 2, n - 2, n - 1};
    for (int k = 0; k < 6 + 32; ++k) {
      const uint64_t h = splitmix64(((uint64_t)n << 6) | (uint64_t)k);
      const int64_t j = k < 6 ? fixed[k] : (int64_t)(h % (uint64_t)n);
      if (j < 0 || j >= n) continue;
      bad += resample_id_rcp_bad(j, n, u12_from_bits((uint32_t)(h >> 32)));
      ++cnt;
    }
  }
  for (int s = 0; s < n_ns; ++s) {
    const int64_t n = ns[s];
#ifdef _OPENMP
#pragma omp parallel for reduction(+ : bad, cnt) schedule(static)
#endif
    for (int64_t j = 0; j < n; ++j) {
      const uint64_t h = splitmix64((uint64_t)j ^ ((uint64_t)n << 32));
      bad += resample_id_rcp_bad(j, n, u12_from_bits((uint32_t)h));
      ++cnt;
    }
#ifdef _OPENMP
#pragma omp parallel for reduction(+ : bad, cnt) schedule(static)
#endif
    for (int64_t m = 0; m < ((int64_t)1 << 23); ++m) {
      const int64_t j = (int64_t)(splitmix64((uint64_t)m + ((uint64_t)n << 24)) % (uint64_t)n);
      bad += resample_id_rcp_bad(j, n, u12_from_bits((uint32_t)m));
      ++cnt;
    }
  }
  if (evaluated) *evaluated = cnt;
  return bad;
}

/* raw Philox4x32-10 block (for the known-answer vectors of the Random123 distribution) */
void crb_oracle_philox4x32(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]) {
  uint32_t c[4] = {ctr[0], ctr[1], ctr[2], ctr[3]};
  uint32_t k[2] = {key[0], key[1]};
  for (int r = 0; r < 10; ++r) {
    philox_round(c, k);
    k[0] += 0x9E3779B9u;
    k[1] += 0xBB67AE85u;
  }
  for (int i = 0; i < 4; ++i) out[i] = c[i];
}

/* ---- resampling() + cumsum(): src/particle_filter.cpp:111-148 ----------------------------------------
 * px [4][n] SoA, pw [n], uniforms [n]: the uni_d(gen) draws in [1,2) (:242), in particle order.
 * reference_mode = 1 reproduces the reference's float arithmetic exactly (float dot product for Neff,
 * float sequential cumsum of pw and of Ones*1.0/NP for `base`); reference_mode = 0 is the batched engine's
 * statement (sum of squares and cumulative sum accumulated in double, base(j) = j/n), which is what makes
 * sense for 10^6 particles.  Returns 1 when resampling happened (Neff < nth). */
int crb_oracle_pf_resample(int64_t n, float* px, float* pw, const double* uniforms, float nth,
                           int reference_mode, float* neff_out) {
  float neff;
  if (reference_mode) {
    float dot = pw[0] * pw[0];
    for (int64_t i = 1; i < n; ++i) dot = dot + pw[i] * pw[i];
    neff = (float)(1.0 / (double)dot);                                   /* :126 */
  } else {
    double dot = 0.0;
    for (int64_t i = 0; i < n; ++i) dot += (double)pw[i] * (double)pw[i];
    neff = (float)(1.0 / (double)(float)dot);
  }
  if (neff_out) *neff_out = neff;
  if (!(neff < nth)) return 0;                                           /* :127 */
  float* wcum = (float*)malloc((size_t)n * sizeof(float));
  float* base = (float*)malloc((size_t)n * sizeof(float));
  float* out = (float*)malloc((size_t)4 * n * sizeof(float));
  if (reference_mode) {
    const float inc = (float)1.0 / (float)n;                             /* Ones()*1.0/NP element */
    wcum[0] = pw[0];
    float c = pw[0] * 0.0f + inc;                                        /* pw*0.0 + Ones*1.0/NP (:130) */
    base[0] = c - inc;
    for (int64_t i = 1; i < n; ++i) {
      wcum[i] = wcum[i - 1] + pw[i];                                     /* cumsum :111-118 */
      c = c + (pw[i] * 0.0f + inc);
      base[i] = c - inc;
    }
  } else {
    double run = 0.0;
    for (int64_t i = 0; i < n; ++i) {
      run += (double)pw[i];
      wcum[i] = (float)run;
      base[i] = (float)((double)i / (double)n);
    }
  }
  int64_t ind = 0;
  for (int64_t i = 0; i < n; ++i) {
    const float rid = (float)((double)base[i] + uniforms[i] / (double)n); /* :133 */
    while (rid > wcum[ind] && ind < n - 1) ind += 1;                     /* :136-138 */
    for (int f = 0; f < 4; ++f) out[f * n + i] = px[f * n + ind];        /* :139 */
  }
  memcpy(px, out, (size_t)4 * n * sizeof(float));                        /* :145 */
  const float wn = reference_mode ? (float)1.0 / (float)n : (float)(1.0 / (double)n);
  for (int64_t i = 0; i < n; ++i) pw[i] = wn;                            /* :146 */
  free(wcum); free(base); free(out);
  return 1;
}

/* the uniform the CUDA kernel draws when uniforms == NULL: Philox4x32-10(seed, j), counter word 2 tagged */
double crb_oracle_philox_uniform12(uint64_t seed, uint64_t index) {
  uint32_t c[4] = {(uint32_t)index, (uint32_t)(index >> 32), 0x5EED5EEDu, 0u};
  uint32_t k[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
  for (int r = 0; r < 10; ++r) {
    philox_round(c, k);
    k[0] += 0x9E3779B9u;
    k[1] += 0xBB67AE85u;
  }
  return (double)(1.0f + (float)(c[0] >> 9) * 1.1920928955078125e-07f);
}

/* ---- solve_DARE() + dlqr(): src/lqr_steer_control.cpp:75-96 (nx = 4, nu = 1, scalar R) and
 * src/lqr_speed_steer_control.cpp:85-106 (nx = 5, nu = 2, 2x2 R).  Column-major matrices.
 *   Xn = A^T*X*A - A^T*X*B/(R + B^T*X*B) * B^T*X*A + Q        (:81 / :91, evaluated left to right)
 *   stop when max|Xn - X| < eps (:83 / :93) and return Xn; after maxiter iterations return X (:89 / :99)
 *   K  = 1.0/(B^T*X*B + R) * (B^T*X*A)                        (:94)   [nu = 1]
 *   K  = (B^T*X*B + R).inverse() * (B^T*X*A)                  (:104)  [nu = 2]
 * Plain binary32, separate multiply and add, sequential-k sums (see the file header). */
static void mm_cm(const float* A, int ra, int ca, const float* B, int cb, float* C) {
  matmul(A, ra, ca, B, cb, C, CRB_ORDER_SEQ);
}
int crb_oracle_dlqr(int nx, int nu, const float* A, const float* B, const float* Q, const float* R,
                    int maxiter, float eps, float* K /*nu x nx*/, float* Xout /*nx x nx or NULL*/) {
  float X[25], Xn[25], At[25], Bt[10], M1[25], T1[25], V1[10], V2[10], M2[25], M3[25], T2[25];
  float BtX[10], S[4], Sinv[4];
  const int nn = nx * nx;
  transpose(A, nx, nx, At);
  transpose(B, nx, nu, Bt);
  for (int i = 0; i < nn; ++i) X[i] = Q[i];
  int it = 0, converged = 0;
  for (; it < maxiter; ++it) {
    mm_cm(At, nx, nx, X, nx, M1);          /* A^T*X          */
    mm_cm(M1, nx, nx, A, nx, T1);          /* (A^T*X)*A      */
    mm_cm(M1, nx, nx, B, nu, V1);          /* (A^T*X)*B      */
    mm_cm(Bt, nu, nx, X, nx, BtX);         /* B^T*X          */
    mm_cm(BtX, nu, nx, B, nu, S);          /* (B^T*X)*B      */
    if (nu == 1) {
      const float s = R[0] + S[0];
      for (int i = 0; i < nx; ++i) V2[i] = V1[i] / s;
    } else {
      for (int i = 0; i < 4; ++i) S[i] = R[i] + S[i];
      const float det = S[0] * S[3] - S[1] * S[2];
      const float invdet = 1.0f / det;
      Sinv[0] = S[3] * invdet; Sinv[1] = -S[1] * invdet; Sinv[2] = -S[2] * invdet; Sinv[3] = S[0] * invdet;
      mm_cm(V1, nx, 2, Sinv, 2, V2);
    }
    mm_cm(V2, nx, nu, Bt, nx, M2);         /* (...)*B^T      */
    mm_cm(M2, nx, nx, X, nx, M3);          /* (...)*X        */
    mm_cm(M3, nx, nx, A, nx, T2);          /* (...)*A        */
    float maxerr = 0.0f;
    for (int i = 0; i < nn; ++i) {
      Xn[i] = (T1[i] - T2[i]) + Q[i];
      const float e = fabsf(Xn[i] - X[i]);
      if (i == 0 || e > maxerr) maxerr = e;
    }
    if (maxerr < eps) { for (int i = 0; i < nn; ++i) X[i] = Xn[i]; converged = 1; ++it; break; }
    for (int i = 0; i < nn; ++i) X[i] = Xn[i];
  }
  (void)converged;
  /* dlqr */
  float BtXA[10];
  mm_cm(Bt, nu, nx, X, nx, BtX);
  mm_cm(BtX, nu, nx, B, nu, S);
  mm_cm(BtX, nu, nx, A, nx, BtXA);
  if (nu == 1) {
    const float s2 = S[0] + R[0];
    const float inv = (float)(1.0 / (double)s2);          /* double scalar converted to the matrix scalar */
    for (int j = 0; j < nx; ++j) K[j] = inv * BtXA[j];
  } else {
    for (int i = 0; i < 4; ++i) S[i] = S[i] + R[i];
    const float det = S[0] * S[3] - S[1] * S[2];
    const float invdet = 1.0f / det;
    Sinv[0] = S[3] * invdet; Sinv[1] = -S[1] * invdet; Sinv[2] = -S[2] * invdet; Sinv[3] = S[0] * invdet;
    mm_cm(Sinv, 2, 2, BtXA, nx, K);
  }
  if (Xout) for (int i = 0; i < nn; ++i) Xout[i] = X[i];
  return it;
}

void crb_oracle_dlqr_batched(int64_t n, int nx, int nu, const float* A, const float* B, const float* Q,
                             const float* R, int maxiter, float eps, float* K, float* X, int32_t* iters,
                             int nthreads) {
#ifdef _OPENMP
  if (nthreads <= 0) nthreads = omp_get_max_threads();
#pragma omp parallel for num_threads(nthreads) schedule(dynamic, 256)
#endif
  for (int64_t i = 0; i < n; ++i) {
    float a[25], b[10], k[10], x[25];
    for (int f = 0; f < nx * nx; ++f) a[f] = A[(int64_t)f * n + i];
    for (int f = 0; f < nx * nu; ++f) b[f] = B[(int64_t)f * n + i];
    const int it = crb_oracle_dlqr(nx, nu, a, b, Q, R, maxiter, eps, k, x);
    for (int f = 0; f < nu * nx; ++f) K[(int64_t)f * n + i] = k[f];
    if (X) for (int f = 0; f < nx * nx; ++f) X[(int64_t)f * n + i] = x[f];
    if (iters) iters[i] = it;
  }
}


/* ---- glibc's sinf / cosf, restated (what the CUDA kernels' crb_sincosf_libm executes) -------------------
 * glibc >= 2.28: sysdeps/ieee754/flt-32/s_sinf.c, s_cosf.c, sincosf.h (reduce_fast, sinf_poly),
 * s_sincosf_data.c (__sincosf_table).  Third-party code that is not under /root/reference: the reference
 * reaches it through std::sin / std::cos on floats (src/extended_kalman_filter.cpp:29-33, :41-45;
 * src/particle_filter.cpp:33-37).  Everything is binary64 multiply / add / fused multiply-add with one final
 * rounding to float, so the GPU's FP64 pipe can reproduce it.  Pinned by tests/test_oracle_ekf.py against THIS host's libm (the
 * oracle's EKF / PF restatements keep calling libm itself, like the reference).  |y| >= 120 (reduce_large) is
 * not restated: libm is called. */
static uint32_t ls_abstop12(float x) {
  uint32_t u;
  memcpy(&u, &x, 4);
  return (u >> 20) & 0x7ff;
}
void crb_oracle_libm_sincosf(float y, float* sn, float* cs) {
  /* the -mfma build of glibc's sources (what the ifunc selects on hosts with FMA): every a + b * c is fused */
  const uint32_t top = ls_abstop12(y);
  if (top >= 0x42f) { /* |y| >= 120, inf, nan */
    *sn = sinf(y);
    *cs = cosf(y);
    return;
  }
  double x = (double)y;
  int n = 0;
  if (top >= 0x3f4) { /* |y| >= pi/4: reduce_fast, hpi_inv prescaled by 2^24 */
    const double r = x * 0x1.45F306DC9C883p+23;
    n = ((int32_t)r + 0x800000) >> 24;
    x = fma(-(double)n, 0x1.921FB54442D18p0, x);
  } else if (top < 0x398) { /* |y| < 2^-12 */
    *sn = y;
    *cs = 1.0f;
    return;
  }
  const double x2 = x * x;
  const double sgn = ((n + 1) & 2) ? -1.0 : 1.0; /* sign[n & 3] = {1, -1, -1, 1} */
  const double q = (n & 2) ? -1.0 : 1.0;         /* __sincosf_table[1]: cosine coefficients negated */
  const double xs = x * sgn;
  const double x3 = xs * x2;
  const double s1 = fma(x2, -0x1.994eb3774cf24p-13, 0x1.1107605230bc4p-7);
  const double x7 = x3 * x2;
  const double sp = fma(x3, -0x1.555545995a603p-3, xs);
  const float ps = (float)fma(x7, s1, sp);
  const double x4 = x2 * x2;
  const double c2 = fma(x2, q * 0x1.99343027bf8c3p-16, q * -0x1.6c087e89a359dp-10);
  const double c1 = fma(x2, q * -0x1.ffffffd0c621cp-2, q);
  const double x6 = x4 * x2;
  const double cp = fma(x4, q * 0x1.55553e1068f19p-5, c1);
  const float pc = (float)fma(x6, c2, cp);
  *sn = (n & 1) ? pc : ps;
  *cs = (n & 1) ? ps : pc;
}

/* count of arguments in [lo_bits, hi_bits) (stepping the float's bit pattern by `step`, both signs) on which
 * the restatement and the host libm disagree; out[0] = sin mismatches, out[1] = cos mismatches */
void crb_oracle_libm_sincosf_census(uint32_t lo_bits, uint32_t hi_bits, uint32_t step, int64_t* out) {
  int64_t bs = 0, bc = 0;
  for (uint64_t u = lo_bits; u < hi_bits; u += step) {
    const uint32_t b = (uint32_t)u;
    float f;
    memcpy(&f, &b, 4);
    for (int sg = 0; sg < 2; ++sg) {
      const float y = sg ? -f : f;
      volatile float a = sinf(y), c = cosf(y);
      float ms, mc;
      crb_oracle_libm_sincosf(y, &ms, &mc);
      const float av = a, cv = c;
      bs += memcmp(&av, &ms, 4) != 0;
      bc += memcmp(&cv, &mc, 4) != 0;
    }
  }
  out[0] = bs;
  out[1] = bc;
}
