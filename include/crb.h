/* crb.h — C ABI of the H100 batched small-matrix engine for the CppRobotics hot paths.
 *
 * The reference (onlytailei/CppRobotics) has no plugin / FFI surface: its hot functions are free
 * functions inside executable translation units.  This header therefore *defines* the seam at the
 * function signatures themselves; every entry point names the reference function it replaces.
 *
 *   crb_ekf_step_batched[_host]        <- ekf_estimation()      src/extended_kalman_filter.cpp:64-78
 *                                         (motion_model :22-36, jacobF :38-47, observation_model :50-55,
 *                                          jacobH :57-62 are folded into the same kernel)
 *   crb_ekf_step_many_batched           <- the same, each agent with its own Q, R and DT (the reference takes Q and R
 *                                          per call)
 *   crb_pf_predict_weight_batched[_host] <- pf_localization() particle loop  src/particle_filter.cpp:81-102
 *                                         (motion_model :26-40, gauss_likelihood :53-57)
 *   crb_pf_estimate                     <- pf_localization() tail            src/particle_filter.cpp:104-107
 *                                         (calc_covariance :59-71)
 *   crb_pf_resample                     <- resampling() + cumsum()           src/particle_filter.cpp:111-148
 *   crb_pf_step_many_batched            <- pf_localization() + resampling() per robot, each with its own u and z
 *                                          src/particle_filter.cpp:73-148, :257-271
 *   crb_mpc_solve_batched[_host]        <- mpc_solve() + FG_EVAL            src/model_predictive_control.cpp:188-346
 *   crb_mpc_plant_update_batched        <- update()                          src/model_predictive_control.cpp:69-81
 *   crb_mpc_calc_ref_trajectory_batched <- calc_ref_trajectory() :130-170 + calc_nearest_index() :107-127
 *   crb_mpc_calc_ref_trajectory_many_batched <- the same, each agent on its own course (the reference takes the
 *                                          course per call)
 *   crb_lqr_dlqr_batched                <- solve_DARE() + dlqr()  src/lqr_steer_control.cpp:75-96,
 *                                          src/lqr_speed_steer_control.cpp:85-106
 *   crb_dwa_control_batched             <- dwa_control()         src/dynamic_window_approach.cpp:148-155
 *                                         (calc_dynamic_window :52-60, calc_final_input :115-145 and the costs)
 *   crb_dwa_control_many_batched        <- the same, each robot among its own obstacles (the reference takes ob
 *                                          per call)
 *   crb_dwa_motion_batched              <- motion()              src/dynamic_window_approach.cpp:43-50
 *   crb_dwa_control_fleet_batched,      <- the same two, each robot with its own Config (the reference takes config
 *   crb_dwa_motion_fleet_batched           per call)
 *   crb_mptg_optimize_batched           <- TrajectoryOptimizer::optimizer_traj()  include/trajectory_optimizer.h:53-200
 *                                         (MotionModel::generate_last_state, quadratic_interpolation,
 *                                          update of include/motion_model.h:59-150)
 *   crb_mptg_generate_trajectory_batched <- MotionModel::generate_trajectory()  include/motion_model.h:110-131
 *   crb_slp_sample_states_batched       <- calc_uniform_polar_states() / calc_biased_polar_states() /
 *                                          calc_lane_states()    src/state_lattice_planner.cpp:29-113
 *   crb_slp_search_nearest_batched      <- search_nearest_one_from_lookuptable()  src/state_lattice_planner.cpp:115-135
 *                                         (generate_path :137-155 is this search followed by
 *                                          crb_mptg_optimize_batched with crb_slp_default_params)
 *   crb_grid_box_of_obstacles           <- a_star_planning() / dijkstra_star_planning() :115-140 (cells, box)
 *   crb_grid_obstacle_map               <- calc_obstacle_map()   src/a_star.cpp:48-78, src/dijkstra.cpp
 *   crb_grid_plan_batched               <- a_star_planning()     src/a_star.cpp:110-244 (with calc_final_path
 *                                          :31-45), dijkstra_star_planning()  src/dijkstra.cpp
 *   crb_rrt_plan_batched                <- RRT::planning()       include/rrt.h:75-159 (GetNearestNode :161-174,
 *                                          CollisionCheck :176-181)
 *   crb_rrt_plan_many_batched           <- the same, each query among its own obstacles (the reference's RRT takes
 *                                          ob_list per planner, :72)
 *   crb_lqr_steering_control_batched    <- lqr_steering_control() src/lqr_steer_control.cpp:98-133 (4 states),
 *                                          src/lqr_speed_steer_control.cpp:108-151 (5 states), with
 *                                          calc_nearest_index() :55-73 / :65-83 and solve_DARE() + dlqr() inside
 *   crb_lqr_steering_control_many_batched <- the same, each vehicle on its own course (the reference takes the
 *                                          course per call)
 *   crb_lqr_update_batched              <- update()              src/lqr_steer_control.cpp:136-146,
 *                                          src/lqr_speed_steer_control.cpp:154-164
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

/* A noise model per agent: ekf_estimation(xEst, PEst, z, u, Q, R) takes Q and R per call, and robots with different
 * sensors, drive trains or filter periods each have their own.  A model is one crb_ekf_params record (88 bytes: dt at
 * offset 0, Q at 8, R at 72); a model table is a DEVICE array of n_models such records in this struct's own layout,
 * so a std::vector<crb_ekf_params> is copied up as it is.  model_of [n] (int32, device) names each agent's model.
 *
 * crb_ekf_step_many_batched: x, P, z, u and n_steps as in crb_ekf_step_batched; agent i uses models[model_of[i]] for
 * all n_steps steps of the launch, and its x and P are bitwise those of crb_ekf_step_batched run with
 * prm = &models[model_of[i]] (also signed zeros, NaN and inf).  status [n] (device) is optional: NULL is not written.
 * An index outside [0, n_models) reads no record: that agent's x and P are written NaN (a filter whose step did not
 * run must not look as if it had, also when status is NULL) and its status is CRB_EKF_BAD_MODEL; other agents are
 * unaffected.  Host arguments are checked before any device work: a NULL ctx, n < 0, n_steps < 1, n_models < 1,
 * or (n > 0) a NULL x, P, z, u, models or model_of is CRB_ERR_INVALID_ARG; n = 0 is a no-op.  The call only enqueues
 * on the context's stream and can be captured in a CUDA graph.
 *
 * crb_ekf_track_step_many: crb_ekf_track_step with the model table in place of prm (z_host, u_host, x_out_host,
 * async and the two-deep rotation as there).  models, model_of and status are DEVICE arrays that the caller uploads
 * once and reuses every tick.  The track runs on the context's pipeline streams, not its main stream, so the table
 * and model_of must be complete on the device before the call (e.g. after crb_sync), and status is complete when the
 * step's x_out_host is.
 *
 * Agents are independent: a context with a communicator steps its own shard and makes no collective. */
#define CRB_EKF_OK 0
#define CRB_EKF_BAD_MODEL 1   /* model_of[i] is outside [0, n_models): x and P of agent i are written NaN */
int crb_ekf_step_many_batched(crb_ctx* ctx, int64_t n, float* x, float* P, const float* z, const float* u,
                              const crb_ekf_params* models, int32_t n_models, const int32_t* model_of,
                              int n_steps, int32_t* status);
int crb_ekf_track_step_many(crb_ctx* ctx, crb_ekf_track* trk, const float* z_host, const float* u_host,
                            const crb_ekf_params* models, int32_t n_models, const int32_t* model_of,
                            int32_t* status, float* x_out_host, int async);

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
 * PEst comes from one pass of double moments centred on particle 0 (rank 0's on a sharded filter).  Its accuracy does
 * not depend on the distance from the origin, but it does depend on how far particle 0 lies from the cloud: the
 * cancellation error grows with (that distance / the cloud's spread)^2.  With particle 0 in the cloud each entry is
 * within 1e-6 sqrt(P_rr P_cc) of the float64 two-pass covariance around xEst (tested with 5 cm clouds up to 10^5 m
 * away); a light particle 0 kilometres from a centimetre-wide cloud can exceed that.  All-zero weights give NaN.
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

/* Per-robot status of crb_pf_step_many_batched. */
#define CRB_PF_FLEET_OK 0
#define CRB_PF_FLEET_BAD_OBSERVATIONS 1 /* z_of[r] does not name a list of at most CRB_PF_MAX_LANDMARKS rows inside
                                           [0, n_rows): the robot's result column is NaN and its px, pw and px_next
                                           columns are left as they were */
/* Particles per robot of crb_pf_step_many_batched: the largest power of two whose shared-memory slice (24 bytes per
 * particle plus 1280) fits the 227 KB of one CTA. */
#define CRB_PF_FLEET_MAX_NP 8192
/* crb_pf_step for a fleet: n_robots INDEPENDENT filters of np particles each, one complete iteration of every filter in
 * ONE launch (one warp per robot).  Robot r owns columns [r*np, (r+1)*np) of the field-major arrays; each robot
 * normalises, estimates, decides on resampling (Neff < nth, its own) and resamples with its own particles only.
 *   px [4][n_robots*np], pw [n_robots*np] in/out and px_next [4][n_robots*np] out: as crb_pf_step, per robot
 *   u [2][n_robots]   each robot's control; prm->u is ignored, every other field of prm is shared by the batch
 *   z, n_rows, z_off, n_sets, z_of: each robot's observations in the obstacle store described above
 *                     crb_dwa_control_many_batched, k = 3: rows (range, lx, ly) like the reference's z items
 *                     (:263-266), at most CRB_PF_MAX_LANDMARKS rows per list; an empty list means no weight update
 *   noise [2][n_robots*np] or NULL: particle r*np + j then draws Philox4x32-10(seed, r*np + j), the draws
 *                     crb_pf_predict_weight_batched makes for that particle of the whole array
 *   uniforms [n_robots*np] in [1, 2) or NULL: Philox(resample_seed, r*np + j); resampleid_j = j/np + U_j/np with
 *                     the running maximum, the cap at np - 1 and pw = 1/np of crb_pf_step
 *   result [CRB_PF_RESULT_LEN][n_robots] (f64, field-major): each robot's crb_pf_step result
 *   status [n_robots] int32 CRB_PF_FLEET_* (optional, NULL = not written)
 * A robot's px, pw and px_next are bitwise those of crb_pf_predict_weight_batched + crb_pf_step's tail run on that
 * robot alone with its u in prm and its list as the landmarks, up to the summation order of the weight sum and the
 * cumulative weights (the reductions run over the robot's particles in a fixed order of their own).  The estimate's
 * moments are centred on the robot's heaviest particle (ties to the lower index; particle 0 when no weight is a
 * number), not on particle 0: its normalised weight is at least 1/np, so it lies within sqrt(np) standard deviations
 * of the mean and the cancellation costs about np 2^-52 of each variance.  PEst is therefore within
 * 1e-6 sqrt(P_rr P_cc) of the float64 two-pass covariance wherever particle 0 and the cloud lie.  A NaN in one
 * list or all-zero weights in one robot make only that robot's outputs NaN.  On a context with a communicator the
 * robots are independent too: there is no collective, each rank steps its own robots as on one GPU.
 * CRB_ERR_INVALID_ARG before any device work unless 1 <= np <= CRB_PF_FLEET_MAX_NP, n_robots >= 0, prm is given,
 * the store passes its host checks and, for n_robots > 0, px, pw, px_next, u and result are given and px != px_next.
 * n_robots = 0 does nothing.  DEVICE pointers; only enqueues (graph-capturable).
 * Replaces: pf_localization(px, pw, xEst, PEst, z, u) + resampling(px, pw) per robot, src/particle_filter.cpp:73-148,
 * :270-271. */
int crb_pf_step_many_batched(crb_ctx* ctx, int64_t n_robots, int32_t np, float* px, float* pw, float* px_next,
                             const float* u, const float* noise, uint64_t seed, const float* z, int64_t n_rows,
                             const int64_t* z_off, int32_t n_sets, const int32_t* z_of, const crb_pf_params* prm,
                             const float* uniforms, uint64_t resample_seed, float nth, double* result,
                             int32_t* status);

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
 * cx[pind+9] without a bounds check (:110); here the search window is clipped to the course, and a target_ind
 * below -9 (a window index at or past 2^31 as the reference's unsigned loop counts) searches nothing.
 * Replaces: calc_ref_trajectory() :130-170 and calc_nearest_index() :107-127. */
int crb_mpc_calc_ref_trajectory_batched(crb_ctx* ctx, int64_t n, int T, const float* state,
                                        const float* cx, const float* cy, const float* cyaw,
                                        const float* sp, int32_t ncourse, float dl,
                                        int32_t* target_ind, float* xref,
                                        const crb_mpc_params* prm);

/* Per-agent status of crb_mpc_calc_ref_trajectory_many_batched. */
#define CRB_MPC_REF_OK 0
#define CRB_MPC_REF_BAD_COURSE 1 /* course_of[i] does not name a course of 1 to INT32_MAX points inside [0, npts):
                                    xref is NaN and target_ind is left as it is */

/* Course store of the *_many_batched entry points: every course's points concatenated.
 *   cx, cy, cyaw, ck, sp [npts]  the courses back to back (npts is int64_t)
 *   course_off [n_courses + 1] int64_t: course c is [course_off[c], course_off[c + 1])
 *   course_of [n] int32_t: the course of each agent; agents may share a course and need not be sorted by it
 * The offsets are device data: each agent's course is checked on the device before any course point is read
 * (0 <= c < n_courses, 0 <= course_off[c] < course_off[c + 1] <= npts, a length that fits in int32); an agent that
 * fails gets its entry point's BAD_COURSE status and nothing outside the arrays is read.  Indices (ind, target_ind)
 * are course-local: they count from the start of the agent's own course, as the reference sees them. */

/* crb_mpc_calc_ref_trajectory_batched with a course per agent (the course store above; no ck).  Each agent's
 * outputs are bitwise those of crb_mpc_calc_ref_trajectory_batched run on its own course, at any target_ind.
 * status [n] int32 CRB_MPC_REF_* is optional (NULL = not written).  CRB_ERR_INVALID_ARG before any device work as
 * crb_mpc_calc_ref_trajectory_batched, and unless n_courses >= 1, npts >= 1 and, for n > 0, course_off and
 * course_of are given.  DEVICE pointers; only enqueues (graph-capturable). */
int crb_mpc_calc_ref_trajectory_many_batched(crb_ctx* ctx, int64_t n, int T, const float* state, const float* cx,
                                             const float* cy, const float* cyaw, const float* sp,
                                             const int64_t* course_off, int32_t n_courses, int64_t npts,
                                             const int32_t* course_of, float dl, int32_t* target_ind, float* xref,
                                             int32_t* status, const crb_mpc_params* prm);

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
 *   min(2 fl(max_accel dt) + ulp(Mv), max_speed - min_speed) / dv + 2      <= CRB_DWA_MAX_SPEED_SAMPLES
 *   min(2 fl(max_dyawrate dt) + ulp(Mw), 2 max_yawrate) / dw + 2           <= CRB_DWA_MAX_YAWRATE_SAMPLES
 *   rollout steps (the reference's `time += dt` loop, :67-72)              <= CRB_DWA_MAX_STEPS
 * otherwise CRB_ERR_INVALID_ARG.  Here Mv = max(|min_speed|, |max_speed|), Mw = |max_yawrate|, ulp is the float
 * spacing at a magnitude, and dv = v_reso - ulp(Mv + v_reso) / 2, dw = yawrate_reso - ulp(Mw + yawrate_reso) / 2
 * must be > 0.  A window is sampled by the reference's float accumulation (:126-127), whose every sum rounds to
 * at least dv (dw) above the last sample, so for any state it takes fewer samples than the cap and ends. */
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

/* Obstacle store of crb_dwa_control_many_batched and crb_rrt_plan_many_batched: every obstacle list's rows back to
 * back, so that each robot or query plans among its own obstacles.
 *   ob [n_rows][k]  the rows (k = 2: ox, oy for DWA; k = 3: x, y, r for RRT); n_rows is int64_t, ob may be NULL when
 *                   n_rows = 0
 *   ob_off [n_sets + 1] int64_t: list s is rows [ob_off[s], ob_off[s + 1])
 *   ob_of [n] int32_t: the list of each robot or query; lists may be shared, and robots need not be sorted by list
 * Empty lists are valid and mean no obstacles.  The offsets are device data: each robot's reference is checked on the
 * device before any row is read (0 <= s < n_sets, 0 <= ob_off[s] <= ob_off[s + 1] <= n_rows, at most the entry point's
 * per-list cap of rows); one that fails gets its entry point's BAD_OBSTACLES status, and nothing outside the arrays is
 * read.  CRB_ERR_INVALID_ARG before any device work unless n_sets >= 1, n_rows >= 0 and, for n > 0, ob_off and ob_of
 * are given and ob is given unless n_rows = 0. */

/* Per-robot status of crb_dwa_control_many_batched. */
#define CRB_DWA_OK 0
#define CRB_DWA_BAD_OBSTACLES 1 /* ob_of[i] does not name a list of at most CRB_DWA_MAX_OBSTACLES rows inside
                                   [0, n_rows): u, cost and traj are NaN and best is -1 */

/* crb_dwa_control_batched with an obstacle list per robot (the obstacle store above, k = 2, at most
 * CRB_DWA_MAX_OBSTACLES rows per list).  Each robot's u, cost, best and traj are bitwise those of
 * crb_dwa_control_batched run with its own list.  status [n] int32 CRB_DWA_* is optional (NULL = not written).
 * CRB_ERR_INVALID_ARG before any device work as crb_dwa_control_batched and for the store's host checks.  One warp
 * per robot, each staging its robot's list in shared memory.  DEVICE pointers; only enqueues (graph-capturable).
 * Replaces: dwa_control(x, u, config, goal, ob) :148-155, which takes its obstacles per call. */
int crb_dwa_control_many_batched(crb_ctx* ctx, int64_t n, const float* x, float* u, const float* goal,
                                 const float* ob, int64_t n_rows, const int64_t* ob_off, int32_t n_sets,
                                 const int32_t* ob_of, const crb_dwa_params* prm, float* cost, int32_t* best,
                                 float* traj, int32_t* status);
/* x [5][n] in/out, u [2][n] (DEVICE; NULL allowed when n = 0).  dt finite and > 0.
 * Replaces: motion(x, u, dt) :43-50, the plant step of main() :194. */
int crb_dwa_motion_batched(crb_ctx* ctx, int64_t n, float* x, const float* u, float dt);

/* A Config per robot: dwa_control(x, u, config, goal, ob) takes its Config per call, and a fleet that mixes robot
 * types has one per type.  A config table is a DEVICE array of n_configs crb_dwa_params records in this struct's own
 * layout (12 floats, 48 bytes, max_speed at offset 0 ... speed_cost_gain at 44), so a std::vector<crb_dwa_params> is
 * copied up as it is.  config_of [n] (int32, device) names each robot's record.
 *
 * crb_dwa_control_fleet_batched: x, u, goal and the obstacle store (k = 2) as in crb_dwa_control_many_batched.  Each
 * record is checked on the device against the limits above, by the same function crb_dwa_rollout_points uses, and
 * n_pts_i = crb_dwa_rollout_points(&configs[config_of[i]]).  For a robot whose record and list are good
 * (CRB_DWA_OK), u, cost and best are bitwise those of crb_dwa_control_many_batched run with prm =
 * &configs[config_of[i]] (best indexes the robot's own grid), and
 *   traj [5*max_pts][n]  gets the first min(n_pts_i, max_pts) points of that call's traj (NaN when best = -1); rows
 *                        past them are not written
 *   traj_len [n]         int32 n_pts_i
 * status [n] int32 CRB_DWA_*.  The config is checked before the list: CRB_DWA_BAD_CONFIG (u and cost NaN, best -1,
 * traj_len 0, traj not written, nothing of the obstacle store read); then CRB_DWA_BAD_OBSTACLES (u and cost NaN,
 * best -1, the first min(n_pts_i, max_pts) points of traj NaN, traj_len n_pts_i).  Other robots are unaffected.
 * cost, best, traj, traj_len and status are optional (NULL = not written).  CRB_ERR_INVALID_ARG before any device
 * work as crb_dwa_control_many_batched (without prm), unless n_configs >= 1, configs and config_of are given when
 * n > 0, and 0 <= max_pts <= CRB_DWA_MAX_STEPS + 1.  n = 0 is a no-op.  One warp per robot; only enqueues
 * (graph-capturable).
 * Replaces: dwa_control(x, u, config, goal, ob) :148-155 with each robot's own config and ob.
 *
 * crb_dwa_motion_fleet_batched: crb_dwa_motion_batched with dt [n] (float, DEVICE) per robot: robot i is bitwise
 * crb_dwa_motion_batched with dt[i].  dt is applied as given (NaN, 0 and negative included), as motion() does.
 * x, u and dt may be NULL when n = 0.
 * Replaces: motion(x, u, config.dt) :43-50 with each robot's config. */
#define CRB_DWA_BAD_CONFIG 2 /* config_of[i] is outside [0, n_configs), or its record is outside the limits above
                                (crb_dwa_rollout_points refuses it) */
int crb_dwa_control_fleet_batched(crb_ctx* ctx, int64_t n, const float* x, float* u, const float* goal,
                                  const float* ob, int64_t n_rows, const int64_t* ob_off, int32_t n_sets,
                                  const int32_t* ob_of, const crb_dwa_params* configs, int32_t n_configs,
                                  const int32_t* config_of, int32_t max_pts, float* cost, int32_t* best, float* traj,
                                  int32_t* traj_len, int32_t* status);
int crb_dwa_motion_fleet_batched(crb_ctx* ctx, int64_t n, float* x, const float* u, const float* dt);

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

/* ---- grid A* and Dijkstra (src/a_star.cpp, src/dijkstra.cpp) ------------------------------------------------ */
/* Many start / goal queries on one obstacle map.  The two files share one skeleton: obstacles rounded to cells, a
 * box of cells [min, max) on each axis, calc_obstacle_map :48-78, then a best-first search over the eight moves of
 * get_motion_model :99-108 with a std::priority_queue ordered by `left->key > right->key`.  Bit-exact with the
 * reference built for x86-64: the same float / double expressions, and the same pop order, ties included (the
 * libstdc++ binary heap's push / pop / adjust steps are restated, DESIGN.md).
 *
 * Scope.  The reference is defined only for a square box and, for A*, a box with min_x = min_y = 0 (it allocates
 * obmap (ywidth, xwidth) but indexes it [x][y], and indexes A*'s path_cost without the box offset), a start inside
 * the box and a reachable goal (otherwise it calls top() on an empty queue).  This library indexes every per-cell
 * array relative to the box, (x - min_x, y - min_y), which inside that domain is the same computation, and defines
 * the rest with the statuses below. */
typedef struct crb_grid_box {
  int32_t min_x, min_y, max_x, max_y; /* cells [min_x, max_x) x [min_y, max_y) */
} crb_grid_box;
/* Box limits: both sides in [1, CRB_GRID_MAX_SIDE] and W * H <= CRB_GRID_MAX_CELLS (W = max_x - min_x,
 * H = max_y - min_y), so every squared cell distance inside the box is exact in double and a cell index with a
 * 3-bit move fits in 32 bits.  Otherwise CRB_ERR_INVALID_ARG. */
#define CRB_GRID_MAX_SIDE 32768
#define CRB_GRID_MAX_CELLS (1 << 24)
/* Device workspace the planner may hold: slots = min(n, resident threads, CRB_GRID_WS_BUDGET / bytes per slot), at
 * least 1, where a slot is a search's cell state (1 byte per cell), A*'s path costs (4 bytes per cell) and its heap
 * (8 bytes per entry, 8 * W * H + 1 entries: every visited cell pushes at most 8). */
#define CRB_GRID_WS_BUDGET ((size_t)1 << 32)

/* The reference's :115-140 on host arrays (no device needed): every obstacle rounded as (int)round(o * 1.0 / reso)
 * in double, box = (min over x, min over y, max over x, max over y).  As in the reference the extreme obstacle
 * column and row lie outside the box (verify_node rejects x >= max_x).  CRB_ERR_INVALID_ARG when n_obs < 1, reso
 * is not finite and > 0, or an obstacle is non-finite or rounds outside the int range. */
int crb_grid_box_of_obstacles(int64_t n_obs, const float* ox, const float* oy, float reso, crb_grid_box* box);

/* calc_obstacle_map :48-78: map [W*H] uint8 out, 1 = blocked, cell (x, y) at (x - min_x) * H + (y - min_y).  A
 * cell is blocked when some obstacle k has (float)sqrt(pow(ox_k - x, 2) + pow(oy_k - y, 2)) <= rr / reso, the root
 * in double and the threshold a float quotient; obstacles are rounded as in crb_grid_box_of_obstacles (one that
 * rounds to a non-finite value or outside the int range blocks nothing).  ox, oy [n_obs], map: DEVICE pointers;
 * reso finite and > 0, rr finite.  Only enqueues on the context's stream. */
int crb_grid_obstacle_map(crb_ctx* ctx, int64_t n_obs, const float* ox, const float* oy, float reso, float rr,
                          const crb_grid_box* box, uint8_t* map);

#define CRB_GRID_ASTAR 0    /* a_star_planning :110-244 */
#define CRB_GRID_DIJKSTRA 1 /* dijkstra_star_planning */

/* Per-query status of crb_grid_plan_batched. */
#define CRB_GRID_FOUND 0         /* the goal cell was popped */
#define CRB_GRID_NO_PATH 1       /* the open set emptied first (goal unreachable, blocked or outside the box) */
#define CRB_GRID_START_OUTSIDE 2 /* the start cell lies outside the box */
#define CRB_GRID_BAD_POINT 3     /* start or goal is non-finite, or round(p / reso) leaves the int range */
#define CRB_GRID_BAD_MAP 4       /* crb_grid_plan_many_batched: map_of[q] is outside [0, n_maps) or names an invalid
                                    table entry (below); takes precedence over BAD_POINT */

/* a_star_planning / dijkstra_star_planning for n queries on one map (the map of crb_grid_obstacle_map, or any
 * uint8 map in its layout, nonzero = blocked).
 *   sg [4][n] in: (sx, sy, gx, gy); cells are (int)roundf(p / reso), a float quotient
 *   optional outputs, NULL = not written:
 *     path [2*max_pts][n]  field 2k + j = component j (x, y) of point k: calc_final_path :31-45, the goal cell first,
 *                          then its parents down to the start, each (float)cell * reso with no box offset; only the
 *                          first min(path_len, max_pts) points are written, the rest is left as it is
 *     path_len [n]         int32: the full number of points (1 when start == goal)
 *     cost [n]             the popped goal entry's key: A* (path_cost[parent] + step) + h(parent), Dijkstra the sum
 *                          of the steps
 *     n_visited [n]        int32: cells popped while unvisited (start and goal included)
 *     status [n]           int32: CRB_GRID_*; other than FOUND: path_len 0, cost NaN (n_visited counts the cells the
 *                          search visited, 0 for START_OUTSIDE and BAD_POINT)
 * The reference's quirks are kept: A*'s heuristic is taken at the expanded node, not the new one; A* pushes only on
 * a strict decrease of path_cost and Dijkstra pushes every valid unvisited neighbour; duplicates stay in the heap and
 * are dropped when popped; a start on an obstacle is expanded.
 * One thread per query (a search is serial: its pop order is the result); persistent lanes take queries from an
 * atomic counter.  The slots' workspace is a grow-only buffer of the context: the first call at a larger
 * W * H * slots allocates (and synchronises the stream), so it cannot be captured in a CUDA graph; later calls only
 * enqueue (a memset and one kernel) and can.  Growing frees the old buffer, so a graph captured before a call that
 * grew the workspace must not be replayed after it: its kernel would use freed device memory.  Capture again (or
 * make the largest call before capturing).  DEVICE pointers, NULL allowed when n = 0. */
int crb_grid_plan_batched(crb_ctx* ctx, int algo, const crb_grid_box* box, const uint8_t* map, float reso, int64_t n,
                          const float* sg, int max_pts, float* path, int32_t* path_len, float* cost,
                          int32_t* n_visited, int32_t* status);
/* The number of slots (concurrent searches) crb_grid_plan_batched uses for these arguments. */
int crb_grid_plan_slots(crb_ctx* ctx, int algo, const crb_grid_box* box, int64_t n, int64_t* slots);

/* Map table of crb_grid_obstacle_map_many and crb_grid_plan_many_batched: many maps back to back in one byte store,
 * each in crb_grid_obstacle_map's layout, so that every robot or query plans on its own map (its own obstacles,
 * window, resolution or robot radius).
 *   boxes [n_maps]      crb_grid_box of each map
 *   reso [n_maps]       float: each map's resolution
 *   map_off [n_maps + 1] int64_t: map m is bytes [map_off[m], map_off[m + 1]) of maps [n_cells] uint8, cell (x, y) at
 *                       map_off[m] + (x - min_x) * H + (y - min_y), nonzero = blocked
 * Host scalars: n_maps >= 1, n_cells >= 0 and max_cells in [1, CRB_GRID_MAX_CELLS], a bound on W * H of every map the
 * call uses (it sizes the planner's slots, so the host never reads the table).  Entry m is valid when its box is within
 * the box limits above, W * H <= max_cells, 0 <= map_off[m], map_off[m + 1] - map_off[m] == W * H, map_off[m + 1] <=
 * n_cells, and reso[m] is finite and > 0.  The table is device data: each entry is checked on the device before
 * anything it points at is read, and nothing outside a valid entry's bytes is read or written for it.
 * CRB_ERR_INVALID_ARG before any device work for a scalar out of range or a table pointer that is NULL where the call
 * needs it. */

/* Status of each map of crb_grid_obstacle_map_many. */
#define CRB_GRID_MAP_OK 0
#define CRB_GRID_MAP_BAD 1 /* an invalid table entry, a non-finite rr[m], or an ob_of[m] that does not name a list of
                              the obstacle store: the map's bytes are left as they were */

/* calc_obstacle_map for every map of a table in one launch.  Map m is built from list ob_of[m] of an obstacle store
 * (the one described above crb_dwa_control_many_batched, k = 2: rows (ox, oy), no cap on a list's rows) with its own
 * reso[m] and robot radius rr [n_maps] (float); many maps may share one list.  Every valid map is bitwise
 * crb_grid_obstacle_map run on its list, box, reso and rr (the threshold is the float quotient rr[m] / reso[m]),
 * whatever the other entries hold.  map_status [n_maps] int32 CRB_GRID_MAP_* is optional (NULL = not written).
 * CRB_ERR_INVALID_ARG before any device work for the table's and the store's host checks (n_sets >= 1, n_rows >= 0;
 * ob may be NULL only when n_rows = 0, maps only when n_cells = 0).  One block per (map, 256-cell tile).  DEVICE
 * pointers; only enqueues (graph-capturable). */
int crb_grid_obstacle_map_many(crb_ctx* ctx, const float* ob, int64_t n_rows, const int64_t* ob_off, int32_t n_sets,
                               const int32_t* ob_of, const float* rr, const crb_grid_box* boxes, const float* reso,
                               const int64_t* map_off, int32_t n_maps, int64_t n_cells, int64_t max_cells,
                               uint8_t* maps, int32_t* map_status);

/* crb_grid_plan_batched with a map per query: query q plans on map map_of[q] [n] (int32) of the table above, its start
 * and goal rounded with that map's reso and its path points cell * reso[map_of[q]].  Each query's outputs are bitwise
 * those of crb_grid_plan_batched run on its own map (path truncation at max_pts and the untouched tail included).  A
 * query whose map_of[q] is outside [0, n_maps) or names an invalid entry gets CRB_GRID_BAD_MAP, path_len 0, cost NaN
 * and n_visited 0; other queries are unaffected.  The slots are sized for max_cells
 * (crb_grid_plan_many_slots) in the context's workspace that crb_grid_plan_batched uses, with the same graph-capture
 * rules: the first call at a larger max_cells * slots grows it and cannot be captured, later calls can, and a graph
 * captured before a call that grew it must not be replayed after.  CRB_ERR_INVALID_ARG before any device work for an
 * unknown algo, the table's host checks, n or n * max_pts out of range as in crb_grid_plan_batched, a NULL boxes,
 * reso, map_off, map_of or sg with n > 0, a NULL maps with n > 0 and n_cells > 0, or a NULL path with max_pts > 0.
 * DEVICE pointers.  Replaces: a_star_planning(sx, sy, gx, gy, ox, oy, reso, rr) / dijkstra_star_planning(...), which
 * take their map's inputs on every call. */
int crb_grid_plan_many_batched(crb_ctx* ctx, int algo, const crb_grid_box* boxes, const float* reso,
                               const int64_t* map_off, int32_t n_maps, const uint8_t* maps, int64_t n_cells,
                               int64_t max_cells, int64_t n, const int32_t* map_of, const float* sg, int max_pts,
                               float* path, int32_t* path_len, float* cost, int32_t* n_visited, int32_t* status);
/* The number of slots crb_grid_plan_many_batched uses for n queries with this max_cells. */
int crb_grid_plan_many_slots(crb_ctx* ctx, int algo, int64_t max_cells, int64_t n, int64_t* slots);

/* ---- RRT (include/rrt.h) ----------------------------------------------------------------------------------------- */
/* Many seeded start / goal queries on one obstacle list.  RRT::planning :75-159 loops until a new node lies within
 * expand_dis of the goal: goal_gen, a std::mt19937, draws goal_dis (uniform_int_distribution<int>(0, 100)) and, when
 * that exceeds goal_sample_rate, a random point (rand_x, then rand_y, both area_dis(goal_gen), a
 * uniform_real_distribution<float>(rand_min, rand_max)), otherwise the goal; GetNearestNode :161-174 picks the first
 * node with the least (float)(pow(dx, 2) + pow(dy, 2)); the new node lies expand_dis from it towards the sample, at
 * atan2f / cosf / sinf; CollisionCheck :176-181 rejects it when its point lies inside an obstacle (the draws are
 * spent, no node is added).  Bit-exact with the reference built for x86-64 with GCC 13 / libstdc++ and glibc 2.39:
 * the generator and both distributions as libstdc++ computes them, glibc's atan2f / cosf / sinf, the double pow /
 * sqrt, float arithmetic without contraction (DESIGN.md).  goal_gen is seeded from std::random_device in the
 * reference; here query i is the reference after goal_gen.seed(seed[i]). */
typedef struct crb_rrt_params {
  float rand_min, rand_max; /* rand_area {min, max}: the area random points are drawn from */
  float expand_dis;         /* distance from the nearest node to a new node, and the goal tolerance */
  int32_t goal_sample_rate; /* the goal is the sample when goal_dis(goal_gen) <= goal_sample_rate (0..100) */
  int32_t max_iter;         /* loop passes per query, rejected ones included (the reference has no cap) */
} crb_rrt_params;
/* RRT's constructor defaults expand_dis 1.0, goal_sample_rate 5 and max_iter 500 (the reference ignores its
 * max_iter; here it is the cap).  rand_area has no default in the reference: the demo's {-2, 15} (src/rrt.cpp) is
 * filled in. */
void crb_rrt_default_params(crb_rrt_params* p);
/* Limits: rand_min <= rand_max, both finite, expand_dis finite, 1 <= max_iter <= CRB_RRT_MAX_ITER; otherwise
 * CRB_ERR_INVALID_ARG before any device work.  A query keeps its nodes (8 bytes each) and parents (2 bytes each) in
 * shared memory with the generator's state (2496 bytes): at CRB_RRT_MAX_ITER that is 166 KB, within one H100 SM's
 * 227 KB for a block. */
#define CRB_RRT_MAX_ITER 16384

/* Per-query status of crb_rrt_plan_batched. */
#define CRB_RRT_FOUND 0     /* a node was accepted within expand_dis of the goal */
#define CRB_RRT_MAX_ITER_REACHED 1 /* max_iter passes without reaching the goal (the reference keeps looping) */
#define CRB_RRT_BAD_INPUT 2        /* a non-finite start, goal or obstacle value, or a nearest-node search with no winner
                                      (every distance NaN or >= FLT_MAX: the reference reads node_list[-1]) */
#define CRB_RRT_BAD_OBSTACLES 3    /* crb_rrt_plan_many_batched: ob_of[q] does not name a list of at most INT32_MAX / 3
                                      rows inside [0, n_rows); n_nodes, n_iter and path_len are 0 */

/* RRT::planning for n queries.
 *   prm: shared by the batch (host pointer)
 *   ob [n_ob][3] rows (x, y, r): circles shared by the batch (n_ob >= 0; NULL allowed when n_ob = 0)
 *   se [4][n] (sx, sy, gx, gy), seed [n] uint32 (goal_gen.seed(seed[q]))
 *   optional outputs, NULL = not written:
 *     path [2*max_pts][n]  field 2k + j = component j (x, y) of point k of planning()'s result: the goal, then the last
 *                          node and its parents down to, but not including, the start, then the start; only the first
 *                          min(path_len, max_pts) points are written, the rest is left as it is
 *     path_len [n]         int32: the full number of points (0 unless FOUND)
 *     tree [2*max_nodes][n], parent [max_nodes][n]
 *                          node_list in insertion order (node 0 is the start) and each node's parent as an index (-1
 *                          for the start); the first min(n_nodes, max_nodes) nodes are written, also for
 *                          MAX_ITER_REACHED
 *     n_nodes [n]          int32: nodes in node_list (0 for a BAD_INPUT found before the loop)
 *     n_iter [n]           int32: loop passes made, rejected ones included
 *     status [n]           int32: CRB_RRT_*
 * One warp per query: the lanes split the nearest-node scan and the obstacle test, and twist the generator together;
 * persistent warps take queries from an atomic counter.  The first call on a context allocates that counter (4 bytes
 * of device memory, kept until crb_destroy), so it cannot be captured in a CUDA graph; later calls only enqueue (a
 * memset and one kernel) and can.  DEVICE pointers (ob, se, seed may be NULL when n = 0: a no-op). */
int crb_rrt_plan_batched(crb_ctx* ctx, const crb_rrt_params* prm, const float* ob, int32_t n_ob, int64_t n,
                         const float* se, const uint32_t* seed, int32_t max_pts, float* path, int32_t* path_len,
                         int32_t max_nodes, float* tree, int32_t* parent, int32_t* n_nodes, int32_t* n_iter,
                         int32_t* status);
/* crb_rrt_plan_batched with an obstacle list per query (the obstacle store described above
 * crb_dwa_control_many_batched, k = 3, at most INT32_MAX / 3 rows per list).  Each query's outputs are bitwise those of
 * crb_rrt_plan_batched run with its own list and the same seed; a non-finite value in a list makes BAD_INPUT of the
 * queries on that list only.  Every other argument, the launch and its graph-capture rule are as there.
 * CRB_ERR_INVALID_ARG before any device work as crb_rrt_plan_batched and for the store's host checks.
 * Replaces: RRT(start, end, ob_list, ...).planning(), whose constructor takes the obstacles per planner (:72). */
int crb_rrt_plan_many_batched(crb_ctx* ctx, const crb_rrt_params* prm, const float* ob, int64_t n_rows,
                              const int64_t* ob_off, int32_t n_sets, const int32_t* ob_of, int64_t n, const float* se,
                              const uint32_t* seed, int32_t max_pts, float* path, int32_t* path_len, int32_t max_nodes,
                              float* tree, int32_t* parent, int32_t* n_nodes, int32_t* n_iter, int32_t* status);

/* ---- LQR path tracking (src/lqr_steer_control.cpp, src/lqr_speed_steer_control.cpp) ------------------------------- */
/* The per-tick functions of the two LQR programs for a fleet on one course; the caller keeps the loop
 * (closed_loop_prediction is not a function with defined behaviour in the reference: its time never advances).
 * Bit-exact with the reference built for x86-64 with GCC 13 and glibc 2.39: float arithmetic without contraction,
 * the double macros DT, L and MAX_STEER promoting what they touch, YAW_P2P in double, glibc's atan2f in
 * calc_nearest_index, glibc's double atan2 narrowed to float for the feed-forward, glibc's sinf / cosf / tanf in
 * update (DESIGN.md §3.1-3.4). */
typedef struct crb_lqr_track_params {
  double dt;        /* DT: the error-rate divisor, A(0,1) = A(2,3) = (float)dt, B(4,1) (5 states); update's step */
  double wheelbase; /* L: B(3) = v / L, the feed-forward atan2(L * k, 1), update's yaw rate */
  double max_steer; /* MAX_STEER: update clamps delta to [-max_steer, max_steer] */
  float Q[25];      /* state cost, column-major 5x5; the top-left nx x nx block is used: Q(r,c) = Q[r + 5c] */
  float R[4];       /* input cost, column-major 2x2; the top-left nu x nu block is used (R[0] for 4 states) */
  int32_t maxiter;  /* solve_DARE's iteration cap (the reference's 150) */
  float eps;        /* solve_DARE's tolerance on max|Xn - X| (the reference's 0.01f) */
} crb_lqr_track_params;
/* The reference's constants: dt 0.1, wheelbase 0.5, max_steer 45.0/180*M_PI, Q = I, R = I (nx 5) or 1 (nx 4),
 * maxiter 150, eps 0.01f.  nx is 4 or 5 (any other value is treated as 5). */
void crb_lqr_track_default_params(crb_lqr_track_params* p, int nx);

/* Per-vehicle status of crb_lqr_steering_control_batched. */
#define CRB_LQR_TRACK_OK 0
#define CRB_LQR_TRACK_DARE_MAXITER 1 /* solve_DARE stopped at maxiter without max|Xn - X| < eps (always at v = 0);
                                        a flag only: the outputs are the reference's, computed from the last X */
#define CRB_LQR_TRACK_BAD_INDEX 2    /* no course point won the scan (every squared distance NaN or >= FLT_MAX) and
                                        the incoming ind is outside [0, ncourse), where the reference reads out of
                                        bounds: u and K are NaN, iters 0, ind / pe / pth_e are left as they are */
#define CRB_LQR_TRACK_BAD_COURSE 3   /* crb_lqr_steering_control_many_batched: course_of[i] does not name a course
                                        of 1 to INT32_MAX points inside [0, npts): u and K are NaN, iters 0, ind / pe /
                                        pth_e are left as they are */

/* lqr_steering_control for n vehicles against one course shared by the batch.
 *   nx 4: lqr_steer_control.cpp (nu = 1); nx 5: lqr_speed_steer_control.cpp (nu = 2)
 *   state [4][n] (x, y, yaw, v)
 *   cx, cy, cyaw, ck [ncourse]; sp [ncourse] for nx 5 (the target speed), NULL for nx 4
 *   ind [n] int32: nx 4 in/out, the nearest index kept across calls (the reference's int& ind: it is only assigned
 *        when a course point wins the scan); nx 5 out, the nearest index of this call (the reference's local, from 0)
 *   pe, pth_e [n] in/out: the previous lateral and heading errors, replaced by this call's
 *   u [nu][n]: nx 4 delta; nx 5 (ai, delta), the reference's {ai, delta}
 *   optional outputs, NULL = not written: K [nu*nx][n] the gain (column-major nu x nx), iters [n] int32 DARE
 *   iterations, status [n] int32 CRB_LQR_TRACK_*
 * calc_nearest_index scans the WHOLE course with a strict '<' against FLT_MAX, so the first minimum wins, and returns
 * the signed squared distance (negated when YAW_P2P(cyaw[ind] - atan2f(dyl, dxl)) < 0), as the reference does.
 * Non-finite states follow the reference's arithmetic (NaN payloads aside).  One thread per vehicle; each block
 * streams the course through shared memory in tiles.  Returns CRB_ERR_INVALID_ARG before any device work unless
 * nx is 4 or 5, ncourse >= 1, sp is given exactly when nx is 5, and prm is valid (crb_lqr_update_batched's limits,
 * finite Q and R, finite eps, maxiter >= 0).  DEVICE pointers; only enqueues (graph-capturable). */
int crb_lqr_steering_control_batched(crb_ctx* ctx, int64_t n, int nx, const float* state, const float* cx,
                                     const float* cy, const float* cyaw, const float* ck, const float* sp,
                                     int32_t ncourse, const crb_lqr_track_params* prm, int32_t* ind, float* pe,
                                     float* pth_e, float* u, float* K, int32_t* iters, int32_t* status);
/* crb_lqr_steering_control_batched with a course per vehicle: cx, cy, cyaw, ck, sp [npts], course_off and course_of
 * are the course store described above crb_mpc_calc_ref_trajectory_many_batched; every other argument is as there,
 * including the 4-state program's persistent ind and CRB_LQR_TRACK_BAD_INDEX, both against the vehicle's own course.
 * Each vehicle's outputs are bitwise those of crb_lqr_steering_control_batched run on its own course.  Each warp
 * searches one vehicle's course at a time (coalesced loads, a warp argmin that keeps the first minimum), then one
 * thread per vehicle runs the rest.  CRB_ERR_INVALID_ARG before any device work as crb_lqr_steering_control_batched,
 * and unless n_courses >= 1, npts >= 1 and, for n > 0, course_off and course_of are given.  DEVICE pointers; only
 * enqueues (graph-capturable). */
int crb_lqr_steering_control_many_batched(crb_ctx* ctx, int64_t n, int nx, const float* state, const float* cx,
                                          const float* cy, const float* cyaw, const float* ck, const float* sp,
                                          const int64_t* course_off, int32_t n_courses, int64_t npts,
                                          const int32_t* course_of, const crb_lqr_track_params* prm, int32_t* ind,
                                          float* pe, float* pth_e, float* u, float* K, int32_t* iters,
                                          int32_t* status);
/* update(State&, a, delta) of the LQR programs for n vehicles: state [4][n] in/out, a [n], delta [n].  The kinematic
 * bicycle of crb_mpc_plant_update_batched with prm's dt, wheelbase and max_steer used as the doubles they are, and
 * no speed clamp.  Requires finite dt, wheelbase and max_steer with |max_steer| < 120 (the range in which tanf is
 * restated); otherwise CRB_ERR_INVALID_ARG.  DEVICE pointers. */
int crb_lqr_update_batched(crb_ctx* ctx, int64_t n, float* state, const float* a, const float* delta,
                           const crb_lqr_track_params* prm);

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
/* One launch, enqueued on the context's stream, of a kernel with the memory access pattern of
 * crb_ekf_step_batched (same arrays, layout, access width and launch shape) and trivial arithmetic: every field
 * of x and P gets (z[0] + z[1]) + (u[0] + u[1]) of its agent added, in place (device pointers, n_steps = 1; n
 * even and the arrays 8-byte aligned, as the EKF step's two-agent form needs).  Timed next to
 * the EKF step it is the bandwidth ceiling of that access pattern (scripts/ekf_ceiling.py). */
int crb_probe_ekf_pattern(crb_ctx* ctx, int64_t n, float* x, float* P, const float* z, const float* u);

#ifdef __cplusplus
}
#endif
#endif /* CRB_H_ */
