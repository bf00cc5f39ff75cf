/* crb_oracle_mpc.h — CPU restatement of the MPC path (see crb_oracle_mpc.c).  TEST INFRASTRUCTURE ONLY. */
#ifndef CRB_ORACLE_MPC_H_
#define CRB_ORACLE_MPC_H_
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define CRB_ORACLE_MPC_MAX_T 32
#define CRB_ORACLE_MPC_CONVERGED 0
#define CRB_ORACLE_MPC_MAX_ITER 1
#define CRB_ORACLE_MPC_NO_DESCENT 2
#define CRB_ORACLE_MPC_NONFINITE 3

/* Same fields, order and meaning as crb_mpc_params in include/crb.h (kept separate on purpose: the
 * oracle does not include product headers). */
typedef struct crb_oracle_mpc_params {
  float dt, wb, max_steer, max_accel, max_speed, min_speed;
  float w_a, w_delta, w_da, w_ddelta, w_x, w_y, w_yaw, w_v;
  int max_iter;
  float du_th;
  int max_ls;
  float j_tol;
} crb_oracle_mpc_params;

void crb_oracle_sincosf(float x, float* sn, float* cs);
/* one agent: xref [T][4], u_init [T-1][2] rows (delta, a) or NULL; sol in the reference's return
 * layout [x(T) | y(T) | yaw(T) | v(T) | delta(T-1) | a(T-1)]; u0 = (a_0, delta_0) */
void crb_oracle_mpc_solve(int T, const float x0[4], const float* xref, const float* u_init,
                          const crb_oracle_mpc_params* p, float* sol, float u0_out[2],
                          float* cost_out, int32_t* status_out, int32_t* iters_out);
void crb_oracle_mpc_solve_batched(int64_t n, int T, const float* x0, const float* xref,
                                  const float* u_init, const crb_oracle_mpc_params* p, float* sol,
                                  float* u0, float* cost, int32_t* status, int32_t* iters,
                                  int nthreads);
/* update() with the reference's macros, and with k = {MAX_STEER, DT, WB, MAX_SPEED, MIN_SPEED} */
void crb_oracle_plant_update(float st[4], float a, float delta);
void crb_oracle_plant_update_k(float st[4], float a, float delta, const double k[5]);
int crb_oracle_calc_nearest_index(const float st[4], const float* cx, const float* cy, int ncourse,
                                  int pind);
/* calc_ref_trajectory() with the reference's DT, and with any DT */
void crb_oracle_calc_ref_trajectory(const float st[4], const float* cx, const float* cy,
                                    const float* cyaw, const float* sp, int ncourse, float dl, int T,
                                    int* target_ind, float* xref);
void crb_oracle_calc_ref_trajectory_dt(const float st[4], const float* cx, const float* cy,
                                       const float* cyaw, const float* sp, int ncourse, float dl, int T,
                                       int* target_ind, float* xref, double DT);
#ifdef __cplusplus
}
#endif
#endif
