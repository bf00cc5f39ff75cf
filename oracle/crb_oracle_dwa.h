/* crb_oracle_dwa.h — CPU restatement of src/dynamic_window_approach.cpp.  TEST INFRASTRUCTURE ONLY. */
#ifndef CRB_ORACLE_DWA_H_
#define CRB_ORACLE_DWA_H_
#include <stdint.h>

#include "../include/crb.h" /* crb_dwa_params and the CRB_DWA_* caps: the same limits as the kernel */
#ifdef __cplusplus
extern "C" {
#endif

/* glibc's acosf restated (fdlibm's binary32 algorithm, what the kernel's crb_dwa_acosf executes) */
float crb_oracle_libm_acosf(float x);
/* mismatches against the host acosf over the bit patterns [lo_bits, hi_bits), both signs (OpenMP) */
int64_t crb_oracle_libm_acosf_census(uint32_t lo_bits, uint32_t hi_bits);
/* motion :43-50 over x [5][n] in place, u [2][n] */
void crb_oracle_dwa_motion(int64_t n, float* x, const float* u, float dt, int nthreads);
/* dwa_control :148-155 with the libcrb layout and outputs of crb_dwa_control_batched (host pointers);
 * nthreads <= 0 means all cores */
void crb_oracle_dwa_control(int64_t n, const float* x, float* u, const float* goal, const float* ob, int n_ob,
                            const crb_dwa_params* c, float* cost, int32_t* best, float* traj, int nthreads);

#ifdef __cplusplus
}
#endif
#endif
