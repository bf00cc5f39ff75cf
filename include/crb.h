/* crb.h — C ABI of the H100 batched small-matrix engine for the CppRobotics hot paths.
 *
 * The reference (onlytailei/CppRobotics) has no plugin / FFI surface: its hot functions are free
 * functions inside executable translation units.  This header therefore *defines* the seam at the
 * function signatures themselves; every entry point names the reference function it replaces.
 *
 *   crb_ekf_step_batched[_host]        <- ekf_estimation()      src/extended_kalman_filter.cpp:64-78
 *                                         (motion_model :22-36, jacobF :38-47, observation_model :50-55,
 *                                          jacobH :57-62 are folded into the same kernel)
 *   crb_pf_predict_weight_batched[_host] <- pf_localization() particle loop  src/particle_filter.cpp:81-102
 *                                         (motion_model :26-40, gauss_likelihood :53-57)
 *   crb_pf_estimate                     <- pf_localization() tail            src/particle_filter.cpp:104-107
 *                                         (calc_covariance :59-71)
 *   crb_pf_resample                     <- resampling() + cumsum()           src/particle_filter.cpp:111-148
 *   crb_mpc_solve_batched[_host]        <- mpc_solve() + FG_EVAL            src/model_predictive_control.cpp:188-346
 *   crb_mpc_plant_update_batched        <- update()                          src/model_predictive_control.cpp:69-81
 *   crb_mpc_calc_ref_trajectory_batched <- calc_ref_trajectory() :130-170 + calc_nearest_index() :107-127
 *   crb_lqr_dlqr_batched                <- solve_DARE() + dlqr()  src/lqr_steer_control.cpp:75-96,
 *                                          src/lqr_speed_steer_control.cpp:85-106
 *   crb_dwa_control_batched             <- dwa_control()         src/dynamic_window_approach.cpp:148-155
 *                                         (calc_dynamic_window :52-60, calc_final_input :115-145 and the costs)
 *   crb_dwa_motion_batched              <- motion()              src/dynamic_window_approach.cpp:43-50
 *   crb_mptg_optimize_batched           <- TrajectoryOptimizer::optimizer_traj()  include/trajectory_optimizer.h:53-200
 *                                         (MotionModel::generate_last_state, quadratic_interpolation,
 *                                          update of include/motion_model.h:59-150)
 *   crb_mptg_generate_trajectory_batched <- MotionModel::generate_trajectory()  include/motion_model.h:110-131
 *   crb_slp_sample_states_batched       <- calc_uniform_polar_states() / calc_biased_polar_states() /
 *                                          calc_lane_states()    src/state_lattice_planner.cpp:29-113
 *   crb_slp_search_nearest_batched      <- search_nearest_one_from_lookuptable()  src/state_lattice_planner.cpp:115-135
 *                                         (generate_path :137-155 is this search followed by
 *                                          crb_mptg_optimize_batched with crb_slp_default_params)
 *   crb_stats_*                         <- (no reference counterpart) per-GPU summary statistics, the
 *                                          only thing that ever crosses NVLink (one all-gather).
 *
 * Conventions
 *   - Plain C, plain pointers and sizes.  No C++ / torch types.
 *   - All batched arrays are SoA, "field-major": element (field f, agent i) lives at ptr[f*n + i].
 *     Matrices are flattened column-major like Eigen fixed-size matrices: P(r,c) is field r + 4*c.
 *   - Entry points without a suffix take DEVICE pointers and enqueue asynchronously on the context's
 *     stream; `_host` variants take HOST pointers and return after the results are in the caller's
 *     buffers.  When every array of the call is pinned and mapped into the device's address space
 *     (crb_host_alloc, cudaHostAlloc / cudaMallocHost, cudaHostRegister) the EKF and PF kernels run
 *     directly on that memory over PCIe (no staging copy) and the MPC solver stores its results
 *     straight into it; any other host memory is staged through internal device buffers in chunks with
 *     copy/compute overlap.  Both routes give the same bits.  CRB_HOST_ZEROCOPY=0 forces staging.
 *   - Back-to-back EKF / PF step launches on one stream use programmatic dependent launch (the next
 *     launch's prologue overlaps the previous launch's tail; data dependencies are still honoured).
 *     CRB_PDL=0 disables it.
 *   - Return value: CRB_OK (0) or a negative crb_status.  crb_last_error_string() describes the last
 *     failure on the calling thread.  The reference reports no errors at all (IPOPT status is dropped,
 *     src/model_predictive_control.cpp:338-339); the per-agent MPC status word is additional.
 *   - The caller owns every buffer.  A context is bound to one device and one stream and is not
 *     thread-safe; use one context per host thread / per GPU (one process per GPU in this repo).
 *   - There is NO CPU fallback: every compute entry point fails with CRB_ERR_NO_DEVICE when no CUDA
 *     device is usable.
 */
#ifndef CRB_H_
#define CRB_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CRB_ABI_VERSION 2

typedef enum crb_status {
  CRB_OK = 0,
  CRB_ERR_INVALID_ARG = -1,
  CRB_ERR_NO_DEVICE = -2,
  CRB_ERR_CUDA = -3,
  CRB_ERR_ALLOC = -4,
  CRB_ERR_UNSUPPORTED = -5
} crb_status;

typedef struct crb_ctx crb_ctx;

/* ---- context ----------------------------------------------------------------------------- */
int crb_abi_version(void);
const char* crb_last_error_string(void);
/* device_id < 0 -> current device.  Creates a private non-blocking stream. */
int crb_init(crb_ctx** out, int device_id);
int crb_destroy(crb_ctx* ctx);
/* Enqueue on a caller-provided cudaStream_t (e.g. torch's current stream) instead of the private
 * one.  The handle is used verbatim: NULL is CUDA's legacy default stream, not "none".
 * crb_use_own_stream() goes back to the context's private stream. */
int crb_set_stream(crb_ctx* ctx, void* cuda_stream);
int crb_use_own_stream(crb_ctx* ctx);
void* crb_get_stream(crb_ctx* ctx);
int crb_sync(crb_ctx* ctx);
/* Number of kernels this context has launched since creation (bench.py's gpu_launches). */
int64_t crb_launch_count(crb_ctx* ctx);
/* Pinned, device-mapped host memory for the _host entry points (enables their zero-copy route). */
int crb_host_alloc(void** out, size_t bytes);
int crb_host_free(void* p);
/* Device memory helpers (for callers that do not want to link the CUDA runtime themselves). */
int crb_device_alloc(crb_ctx* ctx, void** out, size_t bytes);
int crb_device_free(crb_ctx* ctx, void* p);
int crb_memcpy_h2d(crb_ctx* ctx, void* dst_dev, const void* src_host, size_t bytes);
int crb_memcpy_d2h(crb_ctx* ctx, void* dst_host, const void* src_dev, size_t bytes);
/* Event timing on the context's stream (so that callers that only know the C ABI can time it). */
int crb_timer_start(crb_ctx* ctx);
int crb_timer_stop_ms(crb_ctx* ctx, float* ms_out); /* synchronises on the stop event */

/* ---- EKF ------------------------------------------------------------------------------------ */
/* Constants that live in main() of the reference: src/extended_kalman_filter.cpp:17 (DT),
 * :142-146 (Q), :149-151 (R).  dt is a double because DT is a double literal in the reference and
 * several entries are computed as (float)(DT * (double)cosf(yaw)).  Q, R column-major. */
typedef struct crb_ekf_params {
  double dt;
  float Q[16];
  float R[4];
} crb_ekf_params;
/* Fills the reference's constants: dt=0.1, Q=diag(0.1^2,0.1^2,(pi/180)^2,0.1^2), R=I. */
void crb_ekf_default_params(crb_ekf_params* p);

/* n agents, n_steps filter steps per launch (state stays in registers between steps).
 *   x [4][n]  in/out   (px, py, yaw, v)
 *   P [16][n] in/out   column-major 4x4
 *   z [n_steps][2][n]  observations
 *   u [n_steps][2][n]  controls (v, yaw-rate)
 * Replaces: ekf_estimation(xEst, PEst, z, u, Q, R), src/extended_kalman_filter.cpp:64-78. */
int crb_ekf_step_batched(crb_ctx* ctx, int64_t n, float* x, float* P, const float* z,
                         const float* u, const crb_ekf_params* prm, int n_steps);
int crb_ekf_step_batched_host(crb_ctx* ctx, int64_t n, float* x, float* P, const float* z,
                              const float* u, const crb_ekf_params* prm, int n_steps);

/* Resident-state tracking: the reference's own time loop (src/extended_kalman_filter.cpp:171-183 keeps
 * xEst, PEst across iterations and receives only z, u per step).  A track owns x [4][n] and P [16][n] in device
 * memory; crb_ekf_track_step runs ONE filter step for all n agents from HOST arrays z [2][n], u [2][n] (16 bytes
 * per update over PCIe instead of the 176 of crb_ekf_step_batched_host; pinned + mapped arrays are read by the
 * kernel in place) and, when x_out_host != NULL, returns x [4][n] to the host (16 bytes per update, copied on a
 * second stream so that it overlaps the next step's kernel).
 *   async = 0: returns when x_out_host is complete.
 *   async = 1: returns after enqueueing; z_host / u_host / x_out_host of this step belong to the library until
 *              crb_ekf_track_sync (or a later synchronous step) returns.  At most two steps' outputs are in
 *              flight; rotate two sets of host buffers.
 * crb_ekf_track_read copies the current x and / or P to the host (synchronises first).  Results are bit-identical
 * to crb_ekf_step_batched with the same inputs. */
typedef struct crb_ekf_track crb_ekf_track;
int crb_ekf_track_open(crb_ctx* ctx, int64_t n, const float* x0_host, const float* P0_host, crb_ekf_track** out);
int crb_ekf_track_step(crb_ctx* ctx, crb_ekf_track* trk, const float* z_host, const float* u_host,
                       const crb_ekf_params* prm, float* x_out_host, int async);
int crb_ekf_track_sync(crb_ctx* ctx, crb_ekf_track* trk);
int crb_ekf_track_read(crb_ctx* ctx, crb_ekf_track* trk, float* x_host, float* P_host);
int crb_ekf_track_close(crb_ctx* ctx, crb_ekf_track* trk);

/* ---- particle filter -------------------------------------------------------------------------- */
/* Constants from src/particle_filter.cpp: DT :18, PI :19 (3.141592653, *not* M_PI), Q :217 (0.01),
 * Rsim :228-230.  rsim_diag are the two diagonal entries Rsim(0,0), Rsim(1,1) used at :87-88. */
typedef struct crb_pf_params {
  double dt;
  double pi;       /* the reference's truncated PI literal */
  float Q;         /* observation variance; sigma = sqrtf(Q) (:98) */
  float rsim_diag[2];
  float u[2];      /* shared control input */
} crb_pf_params;
void crb_pf_default_params(crb_pf_params* p);

#define CRB_PF_MAX_LANDMARKS 64
/*   px [4][n] in/out particles, pw [n] in/out weights
 *   noise [2][n] standard-normal draws g1,g2 (the reference draws them as doubles from
 *         std::normal_distribution<>, :87-88; here they are explicit f32 inputs), or NULL to draw
 *         them in-kernel from Philox4x32-10(seed, particle index) + Box-Muller.
 *   landmarks [n_lm][3] rows (range, lx, ly) exactly like the reference's z items (:263-266);
 *         HOST pointer in both variants (tiny, copied to constant memory).
 * Replaces: the particle loop of pf_localization, src/particle_filter.cpp:81-102. */
int crb_pf_predict_weight_batched(crb_ctx* ctx, int64_t n, float* px, float* pw,
                                  const float* noise, uint64_t seed, const float* landmarks,
                                  int n_lm, const crb_pf_params* prm);
int crb_pf_predict_weight_batched_host(crb_ctx* ctx, int64_t n, float* px, float* pw,
                                       const float* noise, uint64_t seed, const float* landmarks,
                                       int n_lm, const crb_pf_params* prm);
/* Normalise weights, weighted mean and covariance (device pointers; outputs are HOST pointers).
 *   pw is normalised in place (pw / pw.sum(), :104); xEst[4] = px * pw (:106);
 *   PEst[16] (column-major) = sum_i pw_i (px_i - xEst)(px_i - xEst)^T (:59-71, :107).
 * Reductions are done in double on the device (deterministic two-pass tree), so results are
 * independent of the launch geometry.  sum_w_out (optional) receives the pre-normalisation sum.
 * On a context with a communicator (particles sharded over GPUs) the sums run over ALL ranks (two small
 * all-reduces): every rank normalises by the global weight sum and gets the global estimate.
 * Weights whose exponent underflows are floored at w * 2^-126 by the default predict+weight kernel (the
 * reference's running float product would go denormal or 0): if EVERY particle is far from the observations the
 * reference divides 0 / 0 (:104) whereas this engine returns uniform weights - watch sum_w. */
int crb_pf_estimate(crb_ctx* ctx, int64_t n, const float* px, float* pw, float* xEst_host,
                    float* PEst_host, double* sum_w_out_host);

/* Low-variance resampling when the effective particle count drops (device pointers).
 *   Neff = 1 / sum(pw^2); if Neff < nth (the reference's NTh = NP/2, :22): cumulative weights, one
 *   uniform draw per particle in [1,2) (the reference's uni_d, :242 - the offset by 1/NP is its quirk),
 *   resampleid_j = j/NP + U_j/NP (:133), for each j the first index whose cumulative weight reaches it,
 *   capped at NP-1 (:136-143), gather, and pw = 1/NP (:147).  px is updated in place (px_tmp [4][n] is
 *   workspace).  uniforms [n] are explicit inputs in [1,2), or NULL to draw them from Philox4x32-10(seed,
 *   particle index).  The cumulative sum is accumulated in double (the reference sums 100 floats in
 *   float).  *did_resample_host (optional) receives 0/1, *neff_host (optional) Neff.
 * Replaces: resampling() + cumsum(), src/particle_filter.cpp:111-148. */
int crb_pf_resample(crb_ctx* ctx, int64_t n, float* px, float* pw, float* px_tmp,
                    const float* uniforms, uint64_t seed, float nth, int* did_resample_host,
                    double* neff_host);

/* One COMPLETE filter iteration without a host round trip: predict + weight (:81-102), normalise + estimate +
 * covariance (:104-107), Neff (:126) and, DECIDED ON THE DEVICE (:127), low-variance resampling (:128-147).
 *   px [4][n]      in/out: predicted particles (like crb_pf_predict_weight_batched)
 *   pw [n]         in/out: normalised weights, or 1/n after a resampling
 *   px_next [4][n] out: the particles for the next iteration - the resampled set, or a copy of px when
 *                  Neff >= nth.  Ping-pong px / px_next between calls (no device copy, no decision to read back).
 *   noise / seed, landmarks, n_lm, prm: as crb_pf_predict_weight_batched; uniforms / resample_seed, nth: as
 *                  crb_pf_resample
 *   result_dev [CRB_PF_RESULT_LEN] (device, f64): [0..3] xEst, [4..19] PEst (column-major), [20] sum of the
 *                  un-normalised weights, [21] Neff, [22] 1.0 if resampled, [23] sum of squared weights
 * PEst comes from one pass of double moments centred on particle 0 (rank 0's on a sharded filter), so its accuracy
 * does not depend on the distance from the origin: each entry is within 1e-6 sqrt(P_rr P_cc) of the float64
 * two-pass covariance around xEst (tested with 5 cm clouds up to 10^5 m away).  All-zero weights give NaN.
 * Everything is enqueued on the context's stream (capturable in a CUDA graph).  On a context with a communicator
 * (a filter sharded over GPUs) the weight sum and the moments are all-reduced (one 120-byte all-reduce), every
 * rank gets the global xEst / PEst, weights are normalised globally, and particles are NOT resampled (px_next is
 * a copy; [21..23] are not written).  Also fixes round 1's resampling for n that is not a power of two (the
 * running maximum of resampleid, see the kernel).
 * Replaces: pf_localization() + resampling(), src/particle_filter.cpp:73-148. */
#define CRB_PF_RESULT_LEN 24
int crb_pf_step(crb_ctx* ctx, int64_t n, float* px, float* pw, float* px_next, const float* noise,
                uint64_t seed, const float* landmarks, int n_lm, const crb_pf_params* prm,
                const float* uniforms, uint64_t resample_seed, float nth, double* result_dev);

/* ---- MPC -------------------------------------------------------------------------------------- */
/* Problem constants: src/model_predictive_control.cpp:23-48 (macros), cost weights :202-210 and
 * :247-250, bounds :283-301.  T (number of stages incl. the initial state) is a call argument;
 * the reference compiles T=6 (:24), BASELINE configs use T=20. */
typedef struct crb_mpc_params {
  float dt;            /* DT 0.2            :26 */
  float wb;            /* WB 2.5            :36 */
  float max_steer;     /* 45 deg            :27, bounds :288-291 */
  float max_accel;     /* 1.0               :39, bounds :293-296 */
  float max_speed;     /* 55/3.6            :37, bounds :298-301 */
  float min_speed;     /* -20/3.6           :38 */
  float w_a, w_delta;          /* 0.01, 0.01   input cost       :203-204 */
  float w_da, w_ddelta;        /* 0.01, 1.0    input-rate cost  :208-209 */
  float w_x, w_y, w_yaw, w_v;  /* 1, 1, 0.5, 0.5 tracking cost  :247-250 */
  int   max_iter;      /* cap on outer linearise-and-solve iterations; default 50 = the max_iter the
                          reference gives IPOPT (:326).  (MAX_ITER 3 :30 and DU_TH 0.1 :31 are macros the
                          reference defines but never uses.) */
  float du_th;         /* stop when sum_t |du_t| <= du_th; default 1e-4 (converged to the NLP optimum) */
  int   max_ls;        /* step halvings per iteration, default 4: alpha = 1 .. 1/16, then the Gauss-Newton retry
                          (no reference counterpart) */
  float j_tol;         /* also stop when the full step changes the cost by <= j_tol * cost (default 1e-6,
                          i.e. ~16 ulp of the binary32 cost: it cannot be resolved any further) */
} crb_mpc_params;
void crb_mpc_default_params(crb_mpc_params* p);

/* Limits.  Every float parameter finite, dt > 0, wb > 0, 0 < max_steer < pi/2, max_accel >= 0,
 * min_speed <= max_speed, the eight weights, du_th and j_tol >= 0, max_iter and max_ls >= 0; otherwise the solve and
 * the plant step return CRB_ERR_INVALID_ARG before any device work.  calc_ref_trajectory uses (and checks) only dt.
 * The defaults are inside these limits. */

#define CRB_MPC_MAX_T 32
/* Per-agent status word (the reference drops IPOPT's status, :338-339). */
#define CRB_MPC_CONVERGED     0  /* sum|du| <= du_th */
#define CRB_MPC_MAX_ITER      1  /* iteration cap reached */
#define CRB_MPC_NO_DESCENT    2  /* line search found no decrease (already at a stationary point) */
#define CRB_MPC_NONFINITE     3  /* non-finite input or iterate */

/*   x0   [4][n]      (x, y, yaw, v)                        <- State x0                     :255
 *   xref [4*T][n]    field (4*t + k): stage t, component k <- M_XREF traj_ref (col-major)  :52,:255
 *   u_init [2*(T-1)][n] warm start, fields [delta_0..delta_{T-2} | a_0..a_{T-2}], or NULL for the
 *                    reference's cold start (all zeros, :266-269)
 *   sol  [4T+2(T-1)][n] or NULL: the reference's return vector, fields in its order
 *                    [x(T) | y(T) | yaw(T) | v(T) | delta(T-1) | a(T-1)]                   :54-60,:341-345
 *   u0   [2][n] or NULL: (a_0, delta_0), the two values the caller consumes                :376
 *   cost [n] or NULL: objective fg[0] at the returned point                                :199-250
 *   status [n] or NULL: CRB_MPC_*;  iters [n] or NULL: executed outer iterations
 * Replaces: mpc_solve(State x0, M_XREF traj_ref), src/model_predictive_control.cpp:255-346. */
int crb_mpc_solve_batched(crb_ctx* ctx, int64_t n, int T, const float* x0, const float* xref,
                          const float* u_init, const crb_mpc_params* prm, float* sol, float* u0,
                          float* cost, int32_t* status, int32_t* iters);
int crb_mpc_solve_batched_host(crb_ctx* ctx, int64_t n, int T, const float* x0, const float* xref,
                               const float* u_init, const crb_mpc_params* prm, float* sol,
                               float* u0, float* cost, int32_t* status, int32_t* iters);
/* crb_mpc_solve_batched with a scheduling hint per problem: hint [n] (device, int32, may be NULL) is an estimate
 * of the problem's work - in a receding-horizon loop (the caller's loop, :372-378, solves the same vehicle every
 * control step) the `iters` of the agent's previous solve.  The solver is adaptive (3..21 outer iterations on the bench
 * batch); starting the problems with the largest hints first removes most of the tail in which a few late-started
 * long problems run alone (with more than ~6 SM-generations of problems there is no tail and the hint is
 * ignored).  The hint changes the ORDER in which problems start and nothing
 * else: results are bit-identical to crb_mpc_solve_batched for any hint.  hint must not alias iters. */
int crb_mpc_solve_batched_hinted(crb_ctx* ctx, int64_t n, int T, const float* x0, const float* xref,
                                 const float* u_init, const crb_mpc_params* prm, float* sol, float* u0,
                                 float* cost, int32_t* status, int32_t* iters, const int32_t* hint);
/* Plant step on the first control: state [4][n] in/out, u0 [2][n] = (a, delta).
 * Uses prm->max_steer, dt, wb, max_speed, min_speed (required, not NULL).  The reference evaluates this
 * step in double because its constants are double macros (:26-38): a parameter equal to the reference's
 * macro rounded to float is taken as the macro's double value (defaults are bit-identical to the
 * reference), any other value is promoted from float.  The same rule gives calc_ref_trajectory its DT.
 * cos and sin of the yaw (|yaw| < 120) and tan of the clamped steering are restatements of x86-64 glibc's
 * sinf / cosf (its FMA build) and tanf, so the step reproduces the reference's bits on such a host.
 * Replaces: update(State&, float a, float delta), src/model_predictive_control.cpp:69-81. */
int crb_mpc_plant_update_batched(crb_ctx* ctx, int64_t n, float* state, const float* u0,
                                 const crb_mpc_params* prm);
/* Reference-trajectory lookup for every agent against one shared course.
 *   course arrays cx, cy, cyaw, sp: DEVICE pointers, ncourse entries each
 *   state [4][n]; target_ind [n] in/out (int32); xref [4*T][n] out
 * Integer index work is bit-exact with the reference, including its quirks (float-typed index,
 * :109; strict '<' first-minimum tie-break, :115; monotone target_ind, :139).  The reference reads
 * cx[pind+9] without a bounds check (:110); here the search window is clipped to the course.
 * Replaces: calc_ref_trajectory() :130-170 and calc_nearest_index() :107-127. */
int crb_mpc_calc_ref_trajectory_batched(crb_ctx* ctx, int64_t n, int T, const float* state,
                                        const float* cx, const float* cy, const float* cyaw,
                                        const float* sp, int32_t ncourse, float dl,
                                        int32_t* target_ind, float* xref,
                                        const crb_mpc_params* prm);

/* ---- LQR (SURVEY.md §8 row f-4) ------------------------------------------------------------------- */
/* Discrete LQR gain by the reference's fixed-point DARE iteration, one problem per agent.
 *   (nx, nu) = (4, 1): solve_DARE + dlqr of src/lqr_steer_control.cpp:75-96        (scalar R)
 *   (nx, nu) = (5, 2): solve_DARE + dlqr of src/lqr_speed_steer_control.cpp:85-106 (2x2 R)
 *   A [nx*nx][n], B [nx*nu][n]: per-agent, column-major (DEVICE);  Q [nx*nx], R [nu*nu]: shared (DEVICE)
 *   maxiter 150 and eps 0.01 are the reference's constants (:77-78 / :87-88)
 *   K [nu*nx][n] out (column-major nu x nx); X [nx*nx][n] out or NULL; iters [n] out or NULL */
int crb_lqr_dlqr_batched(crb_ctx* ctx, int64_t n, int nx, int nu, const float* A, const float* B,
                         const float* Q, const float* R, int maxiter, float eps, float* K, float* X,
                         int32_t* iters);

/* ---- dynamic window approach (src/dynamic_window_approach.cpp) ------------------------------------ */
/* class Config :25-41: the same members in the same order. */
typedef struct crb_dwa_params {
  float max_speed, min_speed, max_yawrate, max_accel, robot_radius, max_dyawrate;
  float v_reso, yawrate_reso, dt, predict_time, to_goal_cost_gain, speed_cost_gain;
} crb_dwa_params;
/* The reference's values, including its truncated PI (3.141592653, :16):
 * max_yawrate = max_dyawrate = (float)(40.0 * PI / 180.0), yawrate_reso = (float)(0.1 * PI / 180.0). */
void crb_dwa_default_params(crb_dwa_params* p);

/* Limits.  Every parameter must be finite, v_reso, yawrate_reso and dt > 0, and
 *   min(2 max_accel dt, max_speed - min_speed) / v_reso + 2          <= CRB_DWA_MAX_SPEED_SAMPLES
 *   min(2 max_dyawrate dt, 2 max_yawrate) / yawrate_reso + 2         <= CRB_DWA_MAX_YAWRATE_SAMPLES
 *   rollout steps (the reference's `time += dt` loop, :67-72)        <= CRB_DWA_MAX_STEPS
 * otherwise CRB_ERR_INVALID_ARG.  A window is sampled by the reference's float accumulation (:126-127); for a
 * state so large that v + v_reso == v the reference never terminates, here the axis stops at its cap. */
#define CRB_DWA_MAX_OBSTACLES 256
#define CRB_DWA_MAX_SPEED_SAMPLES 64
#define CRB_DWA_MAX_YAWRATE_SAMPLES 512
#define CRB_DWA_MAX_STEPS 1000
/* Points of every rollout (steps + 1): 32 for the defaults.  CRB_ERR_INVALID_ARG for parameters out of the
 * limits above. */
int crb_dwa_rollout_points(const crb_dwa_params* p, int* n_pts);

/*   x [5][n] (x, y, yaw, v, yawrate), goal [2][n], u [2][n] in/out (in: only u[1] is read, :121-122)
 *   ob [n_ob][2] rows (ox, oy) shared by the whole batch (may be NULL when n_ob = 0)
 *   optional outputs, NULL = not written:
 *     cost [n]  the final min_cost (10000 when no sample is admissible)
 *     best [n]  int32: v-major flat index of the chosen sample, or -1
 *     traj [5*n_pts][n]  field 5k+j = component j of point k of the chosen rollout (NaN when best = -1)
 * All DEVICE pointers (x, u, goal may be NULL when n = 0: a no-op).  Bit-exact with the reference: its float sample grid, std::max / std::min, the double
 * pow / sqrt of the goal cost, glibc's sinf / cosf / acosf, and its selection rule `min_cost >= cost`
 * (the last sample in v-major order with the minimum cost wins, a NaN cost never does, u = (0, u[1]) when
 * nothing is admissible).  Only enqueues on the context's stream (capturable in a CUDA graph).
 * Replaces: dwa_control() :148-155 (calc_dynamic_window :52-60, calc_final_input :115-145, calc_trajectory
 * :63-74, calc_obstacle_cost :77-101, calc_to_goal_cost :103-113). */
int crb_dwa_control_batched(crb_ctx* ctx, int64_t n, const float* x, float* u, const float* goal,
                            const float* ob, int n_ob, const crb_dwa_params* prm, float* cost,
                            int32_t* best, float* traj);
/* x [5][n] in/out, u [2][n] (DEVICE; NULL allowed when n = 0).  dt finite and > 0.
 * Replaces: motion(x, u, dt) :43-50, the plant step of main() :194. */
int crb_dwa_motion_batched(crb_ctx* ctx, int64_t n, float* x, const float* u, float dt);

/* ---- model-predictive trajectory generation (include/trajectory_optimizer.h, include/motion_model.h) ---- */
/* Shared by the batch: MotionModel's base_l and ds, and optimizer_traj's max_iter, cost_th and h_step. */
typedef struct crb_mptg_params {
  float base_l, ds;
  int32_t max_iter;
  float cost_th;
  float h_step[3];
} crb_mptg_params;
/* The demo's values (src/model_predictive_trajectory_generator.cpp:19-33): base_l 1.0, ds 0.1, max_iter 100,
 * cost_th 0.1f, h_step {0.2f, 0.005f, 0.005f}. */
void crb_mptg_default_params(crb_mptg_params* p);

/* Limits: every float parameter finite, ds > 0, base_l != 0, h_step[k] > 0, 0 <= max_iter <= CRB_MPTG_MAX_ITER,
 * max_pts >= 0; otherwise CRB_ERR_INVALID_ARG.  A roll-out (the `for (float i = 0; i < horizon; i += horizon/n)`
 * loop, :124, :145) may take at most CRB_MPTG_MAX_STEPS steps. */
#define CRB_MPTG_MAX_ITER 1000
#define CRB_MPTG_MAX_STEPS 16384

/* Per-problem status.  The reference has no status; the last three mark problems it does not define or whose
 * bits this library cannot reproduce, and such a problem stops there instead of returning a different answer.
 *   CRB_MPTG_CONVERGED          cost < cost_th (:110); for generate_trajectory: the roll-out completed
 *   CRB_MPTG_MAX_ITER_REACHED   max_iter updates made without converging (:63, :127)
 *   CRB_MPTG_EMPTY_TRAJ         the nominal roll-out of an iteration has no step (distance <= 0, v < 0, a NaN
 *                               parameter): the reference reads sample_traj.back() of an empty vector (:105)
 *   CRB_MPTG_STEP_CAP           a roll-out needs more than CRB_MPTG_MAX_STEPS steps (the reference's loop stalls
 *                               at i + dt == i, or runs for very long)
 *   CRB_MPTG_OUT_OF_RANGE       a roll-out needs tanf of a finite steering with |kp| >= 120, or starts from a yaw
 *                               that is not in (-120, 120): outside the range where this library's tanf / sinf /
 *                               cosf are proven equal to glibc's */
#define CRB_MPTG_CONVERGED 0
#define CRB_MPTG_MAX_ITER_REACHED 1
#define CRB_MPTG_EMPTY_TRAJ 2
#define CRB_MPTG_STEP_CAP 3
#define CRB_MPTG_OUT_OF_RANGE 4

/* optimizer_traj(max_iter, cost_th, h_step) :53-128 for n independent problems.
 *   state [4][n] (x, y, yaw, v), target [3][n] (x, y, yaw)
 *   param [4][n] in/out (distance, steering_sequence[0..2]); steering_sequence[0] is never changed (:121-123)
 *   optional outputs, NULL = not written:
 *     traj [3*max_pts][n]  field 3k+j = component j (x, y, yaw) of point k of the returned Traj; only the first
 *                          min(traj_len, max_pts) points are written, the rest of the array is left as it is
 *     traj_len [n]         int32: the returned Traj's full size (also when it exceeds max_pts)
 *     cost [n]             the cost of the returned Traj's last point (:108-109)
 *     status [n], iters [n] int32: CRB_MPTG_* and the number of parameter updates made (:121-124)
 *   On each status:
 *     CONVERGED       param as returned; traj / traj_len / cost of the trajectory that converged
 *     MAX_ITER_REACHED param after the last update; traj / traj_len / cost of the roll-out made at the START of
 *                     the last iteration, i.e. of the parameter before that update (the reference's quirk); with
 *                     max_iter = 0 traj_len = 0, cost = NaN and param is unchanged
 *     EMPTY_TRAJ, STEP_CAP, OUT_OF_RANGE
 *                     param and iters as they stood when the problem stopped, traj_len = 0, cost = NaN
 * All DEVICE pointers (state, target, param may be NULL when n = 0: a no-op).  Bit-exact with the reference
 * built for x86-64 with glibc 2.39: float arithmetic without contraction, the std::pow / std::sqrt of the cost
 * and YAW_P2P in double, Eigen's 3x3 cofactor inverse (DESIGN.md), glibc's tanf / sinf / cosf, and the line
 * search's `cost <= mincost` rule (a tie goes to alpha 1.5, a NaN or +inf cost never wins).  Only enqueues on
 * the context's stream (capturable in a CUDA graph). */
int crb_mptg_optimize_batched(crb_ctx* ctx, int64_t n, const float* state, const float* target, float* param,
                              const crb_mptg_params* prm, int max_pts, float* traj, int32_t* traj_len,
                              float* cost, int32_t* status, int32_t* iters);
/* MotionModel::generate_trajectory(p) :110-131 (only prm->base_l and prm->ds are used, all are validated).
 *   state [4][n], param [4][n] in; optional outputs traj [3*max_pts][n] and traj_len [n] as above, last [3][n] =
 *   generate_last_state(p) :133-150 (the start's x, y, yaw for an empty roll-out), status [n].
 *   status CONVERGED (the roll-out completed), STEP_CAP or OUT_OF_RANGE; on the last two traj_len = 0 and
 *   last = NaN.  DEVICE pointers, NULL allowed when n = 0. */
int crb_mptg_generate_trajectory_batched(crb_ctx* ctx, int64_t n, const float* state, const float* param,
                                         const crb_mptg_params* prm, int max_pts, float* traj,
                                         int32_t* traj_len, float* last, int32_t* status);

/* ---- state lattice planner (src/state_lattice_planner.cpp) ------------------------------------------------ */
/* The planner's own settings (:22-24, :144-148) for generate_path's optimizer: base_l = L 1.0, ds = DS 0.1,
 * max_iter 100, cost_th 0.1f, h_step {0.5f, 0.02f, 0.02f}; *v = CONST_V 3.0, the speed of the start state
 * (0, 0, 0, v).  generate_path(states, table, k0) is crb_slp_search_nearest_batched followed by
 * crb_mptg_optimize_batched with these parameters and that start state. */
void crb_slp_default_params(crb_mptg_params* p, float* v);

/* Terminal-state samplers.  The batch shares one kind and one set of integers; every query has its own floats. */
#define CRB_SLP_UNIFORM 0 /* calc_uniform_polar_states :47-56 */
#define CRB_SLP_BIASED 1  /* calc_biased_polar_states :58-99 */
#define CRB_SLP_LANE 2    /* calc_lane_states :101-113 */
typedef struct crb_slp_sampler {
  int32_t kind; /* CRB_SLP_* */
  int32_t nxy;  /* position samples (all kinds) */
  int32_t nh;   /* heading samples (UNIFORM, BIASED) */
  int32_t ns;   /* biased sampler's angle resolution (BIASED) */
  int32_t d;    /* distance to the terminal states (UNIFORM, BIASED; LANE takes a float d per query) */
} crb_slp_sampler;
/* Limits: 1 <= nxy <= CRB_SLP_MAX_NXY; for UNIFORM and BIASED also 1 <= nh <= CRB_SLP_MAX_NH; for BIASED also
 * 0 <= ns <= CRB_SLP_MAX_NS; and states per query (below) <= CRB_SLP_MAX_STATES.  Otherwise CRB_ERR_INVALID_ARG. */
#define CRB_SLP_MAX_NXY 4096
#define CRB_SLP_MAX_NH 1024
#define CRB_SLP_MAX_NS (1 << 20)
#define CRB_SLP_MAX_STATES 65536
/* S, the output slots per query: nxy * nh (UNIFORM), max(nxy - 1, 0) * nh (BIASED: the scan never matches its
 * last position sample), nxy (LANE).  -1 (and the error string) for a sampler outside the limits. */
int crb_slp_states_per_query(const crb_slp_sampler* s);

/* Per-query status of crb_slp_sample_states_batched. */
#define CRB_SLP_OK 0
#define CRB_SLP_OUT_OF_RANGE 1 /* a finite sin / cos argument with |x| >= 120, outside the range where this
                                  library's sinf / cosf are proven equal to glibc's: n_states = 0 */

/* The samplers for n_q queries.
 *   qp [F][n_q] per-query floats (SoA):
 *     UNIFORM: F = 4: a_min, a_max, p_min, p_max
 *     BIASED:  F = 5: goal_angle, a_min, a_max, p_min, p_max
 *     LANE:    F = 5: l_center, l_heading, l_width, v_width, d
 *   target [3][n_q * S] out: state j of query q (x, y, yaw) is column q * S + j, in the reference's order; the
 *     slots from n_states[q] on are NaN
 *   n_states [n_q] int32 out: states the reference returns (UNIFORM nxy * nh, LANE nxy, BIASED data-dependent:
 *     the scan's back-step li = j - 1 can repeat a sample); status [n_q] int32 out (CRB_SLP_*), or NULL
 * Bit-exact with the reference built for x86-64 with glibc 2.39: its float / double mixing expression by
 * expression (DESIGN.md), glibc's sinf / cosf, the biased sampler's FLT_MIN start of cnav_max and sequential float
 * sums.  With nxy = 1 the polar samplers' angle is 0 / 0 (NaN), as in the reference.  DEVICE pointers, NULL allowed
 * when n_q = 0 (target also when S = 0).  Only enqueues on the context's stream. */
int crb_slp_sample_states_batched(crb_ctx* ctx, int64_t n_q, const crb_slp_sampler* s, const float* qp,
                                  float* target, int32_t* n_states, int32_t* status);

/* search_nearest_one_from_lookuptable :115-135 for n targets.
 *   target [3][n] (x, y, yaw); table [rows][6] (x, y, yaw, s, km, kf: lookuptable.csv's columns), rows >= 1
 *   k0 [n] or NULL (= 0): generate_path's p.steering_sequence[0] = k0 (:141)
 *   param [4][n] out, in crb_mptg_optimize_batched's layout: (sqrtf(x*x + y*y), k0, km, kf) of the nearest row
 *   row [n] int32 out or NULL: that row's index
 * The distance is sqrtf((dx*dx + dy*dy) + dyaw*dyaw) with no yaw wrap, and a row wins only when it is strictly
 * nearer than the best so far, starting from FLT_MAX: the first of equally near rows wins and a NaN or inf distance
 * never does.  When no row wins (a NaN target, e.g. the polar samplers' with nxy = 1; the reference then reads
 * csv_file[-1]) row = -1 and param is NaN, so crb_mptg_optimize_batched stops that problem with
 * CRB_MPTG_EMPTY_TRAJ (CRB_MPTG_MAX_ITER_REACHED with traj_len 0 when max_iter = 0).  DEVICE pointers (target,
 * table, param may be NULL when n = 0: a no-op; rows is checked all the same).  Only enqueues on the context's
 * stream. */
int crb_slp_search_nearest_batched(crb_ctx* ctx, int64_t n, const float* target, const float* table, int rows,
                                   const float* k0, float* param, int32_t* row);

/* ---- multi-GPU: communicator owned by the context (NCCL, opened at run time) ---------------------- */
/* The batch shards over GPUs by contiguous agent ranges (one crb_ctx per device, one host thread or process
 * each); the only inter-GPU traffic is crb_gather_stats (one all-gather of CRB_STATS_LEN doubles per rank)
 * and, for a sharded particle filter, the all-reduce inside crb_pf_estimate.  Bootstrap like any NCCL
 * program: rank 0 calls crb_comm_get_unique_id, the CRB_COMM_ID_BYTES bytes travel to every rank by the
 * host's own channel, every rank calls crb_comm_init_rank (collectively).  libnccl is dlopen'ed on first use
 * ($CRB_NCCL_LIB, then "libnccl.so.2"); CRB_ERR_UNSUPPORTED when it cannot be found.  A context without a
 * communicator behaves as world = 1. */
#define CRB_COMM_ID_BYTES 128
int crb_comm_nccl_version(void);   /* e.g. 22809; 0 when no NCCL library could be opened */
int crb_comm_get_unique_id(void* id_out /* CRB_COMM_ID_BYTES bytes */);
int crb_comm_init_rank(crb_ctx* ctx, int world, int rank, const void* id);
int crb_comm_destroy(crb_ctx* ctx);  /* also done by crb_destroy */
int crb_comm_world(crb_ctx* ctx);
int crb_comm_rank(crb_ctx* ctx);
/* all_dev [world][CRB_STATS_LEN] (device, f64) <- every rank's stats_dev [CRB_STATS_LEN], enqueued on the
 * context's stream (capturable in a CUDA graph).  SURVEY §8 b-4: "wraps the NCCL all-gather". */
int crb_gather_stats(crb_ctx* ctx, const double* stats_dev, double* all_dev);
/* In-place sum over ranks of `count` doubles on the device (the PF weight / moment sums). */
int crb_comm_allreduce_sum_f64(crb_ctx* ctx, double* buf_dev, int64_t count);

/* ---- summary statistics (the only inter-GPU payload) ------------------------------------------- */
#define CRB_STATS_LEN 8
/* Reduces a per-agent f32 array (and optional status / iteration arrays) on the device into
 * stats_dev[CRB_STATS_LEN] (device pointer, f64):
 *   [0] sum  [1] min  [2] max  [3] n_nonfinite  [4] n_status_converged  [5] sum_iters
 *   [6] position-weighted checksum  sum_i value_i * ((i0+i) % 251 + 1)  [7] n
 * i0 is the global index of this shard's first agent so that the checksum of a sharded run equals
 * the single-GPU one.  crb_gather_stats all-gathers the 8 doubles across ranks. */
int crb_stats_reduce(crb_ctx* ctx, int64_t n, int64_t i0, const float* values,
                     const int32_t* status, const int32_t* iters, double* stats_dev);

/* ---- measurement aid ---------------------------------------------------------------------------------- */
/* Non-tensor binary32 FMA rate of the context's device at its current clocks, in TFLOP/s (best of 5 launches of
 * a register-only FFMA kernel, synchronous).  The denominator of the MPC / LQR roofline fractions. */
int crb_probe_fp32_peak(crb_ctx* ctx, double* tflops_out);

#ifdef __cplusplus
}
#endif
#endif /* CRB_H_ */
