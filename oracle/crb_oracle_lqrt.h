/* crb_oracle_lqrt.h — CPU checker for the LQR path-tracking functions (libcrb's crb_lqr_steering_control_batched and
 * crb_lqr_update_batched): calc_nearest_index, lqr_steering_control and update of src/lqr_steer_control.cpp and
 * src/lqr_speed_steer_control.cpp restated in C, on the host libm (atan2f, atan2, cosf, sinf, tanf) as the reference
 * calls it, with solve_DARE + dlqr from crb_oracle.c. */
#ifndef CRB_ORACLE_LQRT_H_
#define CRB_ORACLE_LQRT_H_
#include <stdint.h>

/* the layout of include/crb.h's crb_lqr_track_params */
typedef struct crb_oracle_lqrt_params {
  double dt, wheelbase, max_steer;
  float Q[25], R[4];
  int32_t maxiter;
  float eps;
} crb_oracle_lqrt_params;

/* calc_nearest_index :55-73 / :65-83 for one state (x, y, yaw, v): returns the signed squared distance, *ind is
 * assigned only when a point wins the scan.  The caller guarantees *ind is in range when none does. */
float crb_oracle_lqrt_nearest(const float st[4], const float* cx, const float* cy, const float* cyaw, int32_t ncourse,
                              int32_t* ind);
/* crb_lqr_steering_control_batched on the host: the same arguments, layouts and statuses.  OpenMP over vehicles
 * (nthreads 0 = all). */
void crb_oracle_lqrt_control_batched(int64_t n, int nx, const float* state, const float* cx, const float* cy,
                                     const float* cyaw, const float* ck, const float* sp, int32_t ncourse,
                                     const crb_oracle_lqrt_params* p, int32_t* ind, float* pe, float* pth_e, float* u,
                                     float* K, int32_t* iters, int32_t* status, int nthreads);
/* crb_lqr_update_batched on the host: state [4][n] in/out */
void crb_oracle_lqrt_update_batched(int64_t n, float* state, const float* a, const float* delta,
                                    const crb_oracle_lqrt_params* p, int nthreads);
/* the feed-forward (float)atan2(L * (double)k, 1.0) for every k with bit pattern in [lo_bits, hi_bits): mismatches
 * against got [hi_bits - lo_bits] (the device's results), bitwise (OpenMP) */
int64_t crb_oracle_lqrt_ff_check(double L, uint32_t lo_bits, uint32_t hi_bits, const float* got);
#endif
