// crb_dwa.cu — dynamic window approach (dwa_control, motion) for a batch of robots, for sm_90a.
//
// Replaces dwa_control() and motion() of src/dynamic_window_approach.cpp (:43-155) for n independent robots that
// share one obstacle list (crb_dwa_control_kernel) or each have their own (crb_dwa_control_many_kernel).  Bit-exact
// with the reference compiled for x86-64: float arithmetic without contraction (-fmad=false), glibc's sinf / cosf
// (crb_sincosf_libm) and acosf (crb_dwa_acosf), the goal cost's std::pow / std::sqrt in double, and the
// reference's own float accumulation of the sample grid.
//
// Mapping: one warp per robot.  The robot's speed and yaw-rate grids are built into shared memory, the lanes
// stride over the Nv x Ny samples in v-major order, each lane rolls its sample out in registers (only the even
// points and the last one are used, so no trajectory is stored), and a shuffle reduction picks the winner.
// The winning rollout is computed again, by every lane, to write `traj` when it is requested.  All of that is one
// per-robot body, dwa_robot (crb_dwa_common.cuh, shared with crb_dwa_fleet.cu); the two kernels differ only in how
// they stage the obstacles into shared memory.
#include "crb_dwa_common.cuh"

__global__ void __launch_bounds__(DWA_BLOCK)
crb_dwa_control_kernel(int64_t n, const float* __restrict__ xg, float* __restrict__ ug,
                       const float* __restrict__ goalg, const float* __restrict__ obg, int n_ob,
                       crb_dwa_params p, int n_steps, float* __restrict__ costg, int32_t* __restrict__ bestg,
                       float* __restrict__ trajg) {
  __shared__ float2 s_ob[CRB_DWA_MAX_OBSTACLES];
  __shared__ float s_v[DWA_WARPS][CRB_DWA_MAX_SPEED_SAMPLES];
  __shared__ float s_w[DWA_WARPS][CRB_DWA_MAX_YAWRATE_SAMPLES];
  for (int k = threadIdx.x; k < n_ob; k += DWA_BLOCK) s_ob[k] = make_float2(obg[2 * k], obg[2 * k + 1]);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * DWA_WARPS + warp;
  if (i >= n) return;  // whole warps leave together
  dwa_robot<false>(n, i, lane, s_ob, n_ob, s_v[warp], s_w[warp], xg, ug, goalg, p, n_steps, costg, bestg, trajg,
                   nullptr);
}

// dwa_control with an obstacle list per robot (crb.h's obstacle store, checked by crb_obstacle_list): the same body,
// except that each warp stages its own robot's list into its own slice of shared memory, so dwa_min_d2 reads one
// address across the warp (a broadcast).  A robot whose list reference is bad gets NaN u, cost and traj, best -1 and
// CRB_DWA_BAD_OBSTACLES; nothing of the store past ob_of[i] and two offsets is read for it.  With every robot on one
// list this kernel took 7.7 % longer than crb_dwa_control_kernel on an H100 (DESIGN.md §3), so the shared-list entry
// point keeps that kernel.
__global__ void __launch_bounds__(DWA_BLOCK)
crb_dwa_control_many_kernel(int64_t n, const float* __restrict__ xg, float* __restrict__ ug,
                            const float* __restrict__ goalg, const float* __restrict__ obg, int64_t n_rows,
                            const int64_t* __restrict__ ob_off, int32_t n_sets, const int32_t* __restrict__ ob_of,
                            crb_dwa_params p, int n_steps, float* __restrict__ costg, int32_t* __restrict__ bestg,
                            float* __restrict__ trajg, int32_t* __restrict__ statusg) {
  __shared__ float2 s_ob[DWA_WARPS][CRB_DWA_MAX_OBSTACLES];
  __shared__ float s_v[DWA_WARPS][CRB_DWA_MAX_SPEED_SAMPLES];
  __shared__ float s_w[DWA_WARPS][CRB_DWA_MAX_YAWRATE_SAMPLES];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * DWA_WARPS + warp;
  if (i >= n) return;  // whole warps leave together
  int64_t ob0, ob1;
  if (!crb_obstacle_list(i, ob_off, n_sets, ob_of, n_rows, CRB_DWA_MAX_OBSTACLES, ob0, ob1)) {
    const float qnan = __int_as_float(0x7fc00000);
    if (lane == 0) {
      ug[i] = qnan;
      ug[n + i] = qnan;
      if (costg) costg[i] = qnan;
      if (bestg) bestg[i] = -1;
      if (statusg) statusg[i] = CRB_DWA_BAD_OBSTACLES;
    }
    if (trajg)
      for (int f = lane; f < 5 * (n_steps + 1); f += 32) trajg[(int64_t)f * n + i] = qnan;
    return;
  }
  const int n_ob = (int)(ob1 - ob0);
  float2* ob = s_ob[warp];
  for (int k = lane; k < n_ob; k += 32) ob[k] = make_float2(obg[2 * (ob0 + k)], obg[2 * (ob0 + k) + 1]);
  dwa_robot<false>(n, i, lane, ob, n_ob, s_v[warp], s_w[warp], xg, ug, goalg, p, n_steps, costg, bestg, trajg,
                   statusg);
}

__global__ void __launch_bounds__(256)
crb_dwa_motion_kernel(int64_t n, float* __restrict__ xg, const float* __restrict__ ug, float dt) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s[5];
#pragma unroll
  for (int f = 0; f < 5; ++f) s[f] = xg[(int64_t)f * n + i];
  crb_dwa_motion(s, ug[i], ug[n + i], dt);
#pragma unroll
  for (int f = 0; f < 5; ++f) xg[(int64_t)f * n + i] = s[f];
}

// The parameter limits of crb.h (dwa_params_fault, shared with the Config-table kernel); *n_steps = the reference's
// rollout step count.
static int dwa_check_params(const crb_dwa_params* p, int* n_steps) {
  CRB_REQUIRE(p != nullptr, "params is NULL");
  const char* fault = dwa_params_fault(*p, n_steps);
  CRB_REQUIRE(fault == nullptr, fault);
  return CRB_OK;
}

extern "C" {

void crb_dwa_default_params(crb_dwa_params* p) {
  // src/dynamic_window_approach.cpp:16 PI, :27-40 Config's initialisers (double expressions narrowed to float)
  const double pi = 3.141592653;
  p->max_speed = (float)1.0;
  p->min_speed = (float)-0.5;
  p->max_yawrate = (float)(40.0 * pi / 180.0);
  p->max_accel = (float)0.2;
  p->robot_radius = (float)1.0;
  p->max_dyawrate = (float)(40.0 * pi / 180.0);
  p->v_reso = (float)0.01;
  p->yawrate_reso = (float)(0.1 * pi / 180.0);
  p->dt = (float)0.1;
  p->predict_time = (float)3.0;
  p->to_goal_cost_gain = (float)1.0;
  p->speed_cost_gain = (float)1.0;
}

int crb_dwa_rollout_points(const crb_dwa_params* p, int* n_pts) {
  CRB_REQUIRE(n_pts != nullptr, "n_pts is NULL");
  int steps = 0;
  const int rc = dwa_check_params(p, &steps);
  if (rc != CRB_OK) return rc;
  *n_pts = steps + 1;
  return CRB_OK;
}

int crb_dwa_control_batched(crb_ctx* ctx, int64_t n, const float* x, float* u, const float* goal,
                            const float* ob, int n_ob, const crb_dwa_params* prm, float* cost,
                            int32_t* best, float* traj) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(n >= 0 && (n + DWA_WARPS - 1) / DWA_WARPS <= 0x7fffffff, "n out of range");
  CRB_REQUIRE(n == 0 || (x && u && goal), "x, u or goal is NULL");
  CRB_REQUIRE(n_ob >= 0 && n_ob <= CRB_DWA_MAX_OBSTACLES, "n_ob must be in [0, CRB_DWA_MAX_OBSTACLES]");
  CRB_REQUIRE(ob != nullptr || n_ob == 0, "ob is NULL");
  int n_steps = 0;
  int rc = dwa_check_params(prm, &n_steps);
  if (rc != CRB_OK) return rc;
  if ((rc = crb_require_device(__func__)) != CRB_OK) return rc;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  crb_dwa_control_kernel<<<(unsigned)((n + DWA_WARPS - 1) / DWA_WARPS), DWA_BLOCK, 0, ctx->stream>>>(
      n, x, u, goal, ob, n_ob, *prm, n_steps, cost, best, traj);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

int crb_dwa_control_many_batched(crb_ctx* ctx, int64_t n, const float* x, float* u, const float* goal,
                                 const float* ob, int64_t n_rows, const int64_t* ob_off, int32_t n_sets,
                                 const int32_t* ob_of, const crb_dwa_params* prm, float* cost, int32_t* best,
                                 float* traj, int32_t* status) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(n >= 0 && (n + DWA_WARPS - 1) / DWA_WARPS <= 0x7fffffff, "n out of range");
  CRB_REQUIRE(n == 0 || (x && u && goal), "x, u or goal is NULL");
  CRB_REQUIRE(n_sets >= 1 && n_rows >= 0, "n_sets must be >= 1 and n_rows >= 0");
  CRB_REQUIRE(n == 0 || (ob_off && ob_of && (ob || n_rows == 0)), "ob, ob_off or ob_of is NULL");
  int n_steps = 0;
  int rc = dwa_check_params(prm, &n_steps);
  if (rc != CRB_OK) return rc;
  if ((rc = crb_require_device(__func__)) != CRB_OK) return rc;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  crb_dwa_control_many_kernel<<<(unsigned)((n + DWA_WARPS - 1) / DWA_WARPS), DWA_BLOCK, 0, ctx->stream>>>(
      n, x, u, goal, ob, n_rows, ob_off, n_sets, ob_of, *prm, n_steps, cost, best, traj, status);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

int crb_dwa_motion_batched(crb_ctx* ctx, int64_t n, float* x, const float* u, float dt) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(n >= 0 && (n + 255) / 256 <= 0x7fffffff, "n out of range");
  CRB_REQUIRE(n == 0 || (x && u), "x or u is NULL");
  CRB_REQUIRE(finite_pos(dt), "dt must be finite and > 0");
  const int rc = crb_require_device(__func__);
  if (rc != CRB_OK) return rc;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  crb_dwa_motion_kernel<<<crb_grid_for(n, 256), 256, 0, ctx->stream>>>(n, x, u, dt);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

}  // extern "C"
