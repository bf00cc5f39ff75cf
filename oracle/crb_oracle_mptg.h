/* crb_oracle_mptg.h — CPU restatement of include/trajectory_optimizer.h and include/motion_model.h.
 * TEST INFRASTRUCTURE ONLY. */
#ifndef CRB_ORACLE_MPTG_H_
#define CRB_ORACLE_MPTG_H_
#include <stdint.h>

#include "../include/crb.h" /* crb_mptg_params, the CRB_MPTG_* limits and statuses: the same rules as the kernel */
#ifdef __cplusplus
extern "C" {
#endif

/* glibc 2.39's tanf restated (fdlibm's binary32 k_tanf.c after glibc's binary64 reduce_fast), valid for
 * |x| < 120 and for inf / NaN; what the kernels' crb_tanf_libm executes */
float crb_oracle_libm_tanf(float x);
/* mismatches against the host tanf over the bit patterns [lo_bits, hi_bits), both signs (OpenMP) */
int64_t crb_oracle_libm_tanf_census(uint32_t lo_bits, uint32_t hi_bits);
/* mismatches of got[2 * (u - lo_bits) + sign] (another implementation's results, e.g. the device's) against the
 * restatement over the bit patterns [lo_bits, hi_bits), both signs; NaN equals NaN (OpenMP) */
int64_t crb_oracle_libm_tanf_check(uint32_t lo_bits, uint32_t hi_bits, const float* got);

/* Bits of the optional quirks[] output of crb_oracle_mptg_optimize: which reference corner cases a problem met */
#define CRB_ORACLE_MPTG_CONVERGED_AT_0 1   /* the initial parameter already met cost_th */
#define CRB_ORACLE_MPTG_LS_TIE 2           /* the two line-search costs were equal (alpha 1.5 chosen) */
#define CRB_ORACLE_MPTG_LS_NAN 4           /* a line-search cost was NaN */
#define CRB_ORACLE_MPTG_SINGULAR_J 8       /* J's inverse had a non-finite entry */
#define CRB_ORACLE_MPTG_STEPS_OFF_CEIL 16  /* a nominal roll-out's step count was not ceil(distance / ds) */
#define CRB_ORACLE_MPTG_STEER_BEYOND_PIO4 32 /* tanf was evaluated at |kp| > pi/4 */

/* optimizer_traj :53-128 with the layout and outputs of crb_mptg_optimize_batched (host pointers; the same
 * optional arrays may be NULL); quirks [n] optional.  nthreads <= 0 means all cores. */
void crb_oracle_mptg_optimize(int64_t n, const float* state, const float* target, float* param,
                              const crb_mptg_params* p, int max_pts, float* traj, int32_t* traj_len, float* cost,
                              int32_t* status, int32_t* iters, int32_t* quirks, int nthreads);
/* generate_trajectory / generate_last_state :110-150 with the outputs of crb_mptg_generate_trajectory_batched */
void crb_oracle_mptg_generate(int64_t n, const float* state, const float* param, const crb_mptg_params* p,
                              int max_pts, float* traj, int32_t* traj_len, float* last, int32_t* status,
                              int nthreads);

#ifdef __cplusplus
}
#endif
#endif
