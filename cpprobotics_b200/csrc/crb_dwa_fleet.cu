// crb_dwa_fleet.cu — dynamic window approach for a fleet of mixed robot types, for sm_90a: dwa_control with a Config
// per robot (crb_dwa_control_fleet_kernel) and motion with a dt per robot (crb_dwa_motion_fleet_kernel).
//
// The reference's dwa_control(x, u, config, goal, ob) (src/dynamic_window_approach.cpp:148-155) takes its Config on
// every call, and its main loop steps motion(x, u, config.dt) (:43-50).  Here each robot names a record of a device
// table of crb_dwa_params with config_of[i].  The mapping is crb_dwa_control_many_kernel's (crb_dwa.cu): one warp per
// robot, its obstacle list staged into the warp's slice of shared memory, its grids in the warp's rows, and the same
// per-robot body, dwa_robot (crb_dwa_common.cuh).  What differs is the record: every lane loads the robot's 48 bytes
// (the same address across the warp) and decides it with dwa_params_fault, the function the host entry points use
// for their crb_dwa_params argument, so a record is accepted and stepped exactly as crb_dwa_rollout_points would.
#include "crb_dwa_common.cuh"

__global__ void __launch_bounds__(DWA_BLOCK)
crb_dwa_control_fleet_kernel(int64_t n, const float* __restrict__ xg, float* __restrict__ ug,
                             const float* __restrict__ goalg, const float* __restrict__ obg, int64_t n_rows,
                             const int64_t* __restrict__ ob_off, int32_t n_sets, const int32_t* __restrict__ ob_of,
                             const crb_dwa_params* __restrict__ configs, int32_t n_configs,
                             const int32_t* __restrict__ config_of, int max_pts, float* __restrict__ costg,
                             int32_t* __restrict__ bestg, float* __restrict__ trajg, int32_t* __restrict__ traj_leng,
                             int32_t* __restrict__ statusg) {
  __shared__ float2 s_ob[DWA_WARPS][CRB_DWA_MAX_OBSTACLES];
  __shared__ float s_v[DWA_WARPS][CRB_DWA_MAX_SPEED_SAMPLES];
  __shared__ float s_w[DWA_WARPS][CRB_DWA_MAX_YAWRATE_SAMPLES];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * DWA_WARPS + warp;
  if (i >= n) return;  // whole warps leave together
  const float qnan = __int_as_float(0x7fc00000);
  // the config before the obstacle list: a robot with a bad config reads nothing of the store
  const int32_t c = config_of[i];
  crb_dwa_params p;
  int n_steps = 0;
  bool good = c >= 0 && c < n_configs;
  if (good) {
    p = configs[c];
    good = dwa_params_fault(p, &n_steps) == nullptr;
  }
  if (!good) {
    if (lane == 0) {
      ug[i] = qnan;
      ug[n + i] = qnan;
      if (costg) costg[i] = qnan;
      if (bestg) bestg[i] = -1;
      if (traj_leng) traj_leng[i] = 0;
      if (statusg) statusg[i] = CRB_DWA_BAD_CONFIG;
    }
    return;
  }
  int64_t ob0, ob1;
  if (!crb_obstacle_list(i, ob_off, n_sets, ob_of, n_rows, CRB_DWA_MAX_OBSTACLES, ob0, ob1)) {
    if (lane == 0) {
      ug[i] = qnan;
      ug[n + i] = qnan;
      if (costg) costg[i] = qnan;
      if (bestg) bestg[i] = -1;
      if (traj_leng) traj_leng[i] = n_steps + 1;
      if (statusg) statusg[i] = CRB_DWA_BAD_OBSTACLES;
    }
    if (trajg)
      for (int f = lane; f < 5 * min(n_steps + 1, max_pts); f += 32) trajg[(int64_t)f * n + i] = qnan;
    return;
  }
  const int n_ob = (int)(ob1 - ob0);
  float2* ob = s_ob[warp];
  for (int k = lane; k < n_ob; k += 32) ob[k] = make_float2(obg[2 * (ob0 + k)], obg[2 * (ob0 + k) + 1]);
  dwa_robot<true>(n, i, lane, ob, n_ob, s_v[warp], s_w[warp], xg, ug, goalg, p, n_steps, costg, bestg, trajg, statusg,
                  max_pts);
  if (lane == 0 && traj_leng) traj_leng[i] = n_steps + 1;
}

// motion(x, u, dt[i]) :43-50 per robot; dt is applied as given (motion has no precondition on it).
__global__ void __launch_bounds__(256)
crb_dwa_motion_fleet_kernel(int64_t n, float* __restrict__ xg, const float* __restrict__ ug,
                            const float* __restrict__ dtg) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s[5];
#pragma unroll
  for (int f = 0; f < 5; ++f) s[f] = xg[(int64_t)f * n + i];
  crb_dwa_motion(s, ug[i], ug[n + i], dtg[i]);
#pragma unroll
  for (int f = 0; f < 5; ++f) xg[(int64_t)f * n + i] = s[f];
}

extern "C" {

int crb_dwa_control_fleet_batched(crb_ctx* ctx, int64_t n, const float* x, float* u, const float* goal,
                                  const float* ob, int64_t n_rows, const int64_t* ob_off, int32_t n_sets,
                                  const int32_t* ob_of, const crb_dwa_params* configs, int32_t n_configs,
                                  const int32_t* config_of, int32_t max_pts, float* cost, int32_t* best, float* traj,
                                  int32_t* traj_len, int32_t* status) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(n >= 0 && (n + DWA_WARPS - 1) / DWA_WARPS <= 0x7fffffff, "n out of range");
  CRB_REQUIRE(n == 0 || (x && u && goal), "x, u or goal is NULL");
  CRB_REQUIRE(n_sets >= 1 && n_rows >= 0, "n_sets must be >= 1 and n_rows >= 0");
  CRB_REQUIRE(n == 0 || (ob_off && ob_of && (ob || n_rows == 0)), "ob, ob_off or ob_of is NULL");
  CRB_REQUIRE(n_configs >= 1, "n_configs must be >= 1");
  CRB_REQUIRE(n == 0 || (configs && config_of), "configs or config_of is NULL");
  CRB_REQUIRE(max_pts >= 0 && max_pts <= CRB_DWA_MAX_STEPS + 1, "max_pts must be in [0, CRB_DWA_MAX_STEPS + 1]");
  const int rc = crb_require_device(__func__);
  if (rc != CRB_OK) return rc;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  crb_dwa_control_fleet_kernel<<<(unsigned)((n + DWA_WARPS - 1) / DWA_WARPS), DWA_BLOCK, 0, ctx->stream>>>(
      n, x, u, goal, ob, n_rows, ob_off, n_sets, ob_of, configs, n_configs, config_of, max_pts, cost, best, traj,
      traj_len, status);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

int crb_dwa_motion_fleet_batched(crb_ctx* ctx, int64_t n, float* x, const float* u, const float* dt) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(n >= 0 && (n + 255) / 256 <= 0x7fffffff, "n out of range");
  CRB_REQUIRE(n == 0 || (x && u && dt), "x, u or dt is NULL");
  const int rc = crb_require_device(__func__);
  if (rc != CRB_OK) return rc;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  crb_dwa_motion_fleet_kernel<<<crb_grid_for(n, 256), 256, 0, ctx->stream>>>(n, x, u, dt);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

}  // extern "C"
