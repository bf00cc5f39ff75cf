/* crb_oracle.h — CPU restatement of the CppRobotics hot paths.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load
 * this library.  The product (libcrb.so, cpprobotics_b200/) never links or calls it.
 *
 * PARITY PINNING: the reference ships no tests, golden vectors or fixtures (SURVEY.md §4, §8c-6) and
 * cannot be compiled as-is here (Eigen, OpenCV, CppAD, IPOPT absent).  The EKF / PF / MPC-helper
 * restatements below are pinned (tests/test_oracle_vs_ref.py) against the reference's OWN SOURCE
 * FILES compiled unmodified against header shims for the absent third-party libraries
 * (oracle/shim -> oracle/_ref/libref_*.so), plus hand-derived known answers and float64 numpy
 * restatements (tests/golden/).  What stays unpinned: Eigen's real inner-product summation order
 * (selectable here: CRB_ORDER_SEQ / CRB_ORDER_PAIRWISE) and the MPC solve itself (IPOPT is not
 * available; see crb_oracle_mpc.c).
 */
#ifndef CRB_ORACLE_H_
#define CRB_ORACLE_H_
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define CRB_ORDER_SEQ 0      /* ((a0*b0 + a1*b1) + a2*b2) + a3*b3 : Eigen packet path */
#define CRB_ORDER_PAIRWISE 1 /* (a0*b0 + a1*b1) + (a2*b2 + a3*b3) : Eigen scalar redux unroller */

/* ---- EKF: src/extended_kalman_filter.cpp ------------------------------------------------------ */
/* motion_model :22-36 */
void crb_oracle_motion_model(const float x[4], const float u[2], double dt, float out[4]);
/* jacobF :38-47 (column-major 4x4 out) */
void crb_oracle_jacobF(const float x[4], const float u[2], double dt, float jF[16]);
/* ekf_estimation :64-78; P, Q column-major 4x4, R column-major 2x2 */
void crb_oracle_ekf_estimation(float xEst[4], float PEst[16], const float z[2], const float u[2],
                               const float Q[16], const float R[4], double dt, int order);
/* float64 evaluation of the same formulas (cross-check only) */
void crb_oracle_ekf_estimation_f64(double xEst[4], double PEst[16], const double z[2],
                                   const double u[2], const double Q[16], const double R[4],
                                   double dt);
/* batched SoA driver with the libcrb layout (x[4][n], P[16][n], z/u[n_steps][2][n]); nthreads<=0
 * means all cores */
void crb_oracle_ekf_step_batched(int64_t n, float* x, float* P, const float* z, const float* u,
                                 const float* Q, const float* R, double dt, int n_steps, int order,
                                 int nthreads);

/* ---- PF: src/particle_filter.cpp ---------------------------------------------------------------- */
/* gauss_likelihood :53-57 with the reference's PI literal passed in */
float crb_oracle_gauss_likelihood(float x, float sigma, double pi);
/* one particle of the loop :81-102; g[2] are the two normal draws; landmarks rows (range,lx,ly) */
void crb_oracle_pf_particle(float x[4], float* w, const double g[2], const float u[2],
                            const float rsim_diag[2], const float* landmarks, int n_lm, float Q,
                            double dt, double pi);
/* Philox4x32-10 + Box-Muller exactly as the CUDA kernel draws them when noise == NULL */
void crb_oracle_philox_normal2(uint64_t seed, uint64_t index, float g[2]);
void crb_oracle_pf_predict_weight_batched(int64_t n, float* px, float* pw, const float* noise,
                                          uint64_t seed, const float* landmarks, int n_lm,
                                          const float u[2], const float rsim_diag[2], float Q,
                                          double dt, double pi, int nthreads);
/* :104-107 + calc_covariance :59-71 with double accumulators; pw normalised in place */
void crb_oracle_pf_estimate(int64_t n, const float* px, float* pw, float xEst[4], float PEst[16],
                            double* sum_w);

/* resampling() + cumsum() :111-148 (see crb_oracle.c) */
int crb_oracle_pf_resample(int64_t n, float* px, float* pw, const double* uniforms, float nth,
                           int reference_mode, float* neff_out);
double crb_oracle_philox_uniform12(uint64_t seed, uint64_t index);
/* solve_DARE() + dlqr(): lqr_steer_control.cpp:75-96 / lqr_speed_steer_control.cpp:85-106 */
int crb_oracle_dlqr(int nx, int nu, const float* A, const float* B, const float* Q, const float* R,
                    int maxiter, float eps, float* K, float* Xout);
void crb_oracle_dlqr_batched(int64_t n, int nx, int nu, const float* A, const float* B, const float* Q,
                             const float* R, int maxiter, float eps, float* K, float* X, int32_t* iters,
                             int nthreads);
void crb_oracle_philox4x32(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]);
int crb_oracle_num_threads(void);
/* verification aids for arithmetic shortcuts of the CUDA PF kernel (see crb_oracle.c) */
int64_t crb_oracle_check_const_division(float d, uint32_t lo_bits, uint32_t hi_bits);
int64_t crb_oracle_check_ff_product(double pre, uint32_t lo_bits, uint32_t hi_bits);
int64_t crb_oracle_check_resample_id_rcp(int64_t n_max, const int64_t* ns, int n_ns, int64_t* evaluated);

/* glibc's sinf / cosf restated (binary64 polynomial, what the kernels' crb_sincosf_libm executes) */
void crb_oracle_libm_sincosf(float y, float* sn, float* cs);
void crb_oracle_libm_sincosf_census(uint32_t lo_bits, uint32_t hi_bits, uint32_t step, int64_t* out);
#ifdef __cplusplus
}
#endif
#endif
