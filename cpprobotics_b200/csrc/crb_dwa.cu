// crb_dwa.cu — dynamic window approach (dwa_control, motion) for a batch of robots, for sm_90a.
//
// Replaces dwa_control() and motion() of src/dynamic_window_approach.cpp (:43-155) for n independent robots
// that share one obstacle list.  Bit-exact with the reference compiled for x86-64: float arithmetic without
// contraction (-fmad=false), glibc's sinf / cosf (crb_sincosf_libm) and acosf (crb_dwa_acosf below), the goal
// cost's std::pow / std::sqrt in double, and the reference's own float accumulation of the sample grid.
//
// Mapping: one warp per robot.  The robot's speed and yaw-rate grids are built into shared memory, the lanes
// stride over the Nv x Ny samples in v-major order, each lane rolls its sample out in registers (only the even
// points and the last one are used, so no trajectory is stored), and a shuffle reduction picks the winner.
// The winning rollout is computed again, by every lane, to write `traj` when it is requested.
#include <float.h>

#include "crb_common.cuh"

#define DWA_BLOCK 256
#define DWA_WARPS (DWA_BLOCK / 32)

// motion() :43-50: yaw first, then the position with the NEW yaw, two separate float multiplies per axis.
__device__ __forceinline__ void crb_dwa_motion(float (&s)[5], float v, float w, float dt) {
  s[2] = s[2] + w * dt;
  float sn, cs;
  crb_sincosf_libm(s[2], sn, cs);
  s[0] = s[0] + v * cs * dt;
  s[1] = s[1] + v * sn * dt;
  s[3] = v;
  s[4] = w;
}

// glibc's acosf (the reference's std::acos(float), :109).  glibc 2.39 computes it with fdlibm's binary32
// algorithm (e_acosf.c, Sun Microsystems, freely redistributable): a rational approximation in z = x^2 or
// (1 - |x|) / 2 with three branches and, for x > 0.5, sqrtf(z) split at bit 12 so that 2 (df + w) keeps the
// extra precision.  Restated operation for operation; CUDA's own acosf rounds differently on ~5e6 inputs in
// [-1, 1].  |x| > 1 and NaN give NaN (its bits are not specified: a NaN cost never wins the selection).
__device__ __noinline__ float crb_dwa_acosf(float x) {
  const float pi = 3.1415925026e+00f, pio2_hi = 1.5707962513e+00f, pio2_lo = 7.5497894159e-08f;
  const float pS0 = 1.6666667163e-01f, pS1 = -3.2556581497e-01f, pS2 = 2.0121252537e-01f,
              pS3 = -4.0055535734e-02f, pS4 = 7.9153501429e-04f, pS5 = 3.4793309169e-05f;
  const float qS1 = -2.4033949375e+00f, qS2 = 2.0209457874e+00f, qS3 = -6.8828397989e-01f,
              qS4 = 7.7038154006e-02f;
  const int hx = __float_as_int(x);
  const int ix = hx & 0x7fffffff;
  if (ix == 0x3f800000) return hx > 0 ? 0.0f : pi + 2.0f * pio2_lo;  // |x| == 1
  if (ix > 0x3f800000) return (x - x) / (x - x);                      // |x| > 1, inf, NaN
  if (ix < 0x3f000000) {                                               // |x| < 0.5
    if (ix <= 0x23000000) return pio2_hi + pio2_lo;
    const float z = x * x;
    const float p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
    const float q = 1.0f + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
    const float r = p / q;
    return pio2_hi - (x - (pio2_lo - x * r));
  }
  if (hx < 0) {  // x < -0.5
    const float z = (1.0f + x) * 0.5f;
    const float p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
    const float q = 1.0f + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
    const float s = sqrtf(z);
    const float r = p / q;
    const float w = r * s - pio2_lo;
    return pi - 2.0f * (s + w);
  }
  const float z = (1.0f - x) * 0.5f;  // x > 0.5
  const float s = sqrtf(z);
  const float df = __int_as_float(__float_as_int(s) & (int)0xfffff000);
  const float c = (z - df * df) / (s + df);
  const float p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
  const float q = 1.0f + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
  const float r = p / q;
  const float w = r * s + c;
  return 2.0f * (df + w);
}

// Smallest squared distance from (px, py) to the obstacles, folded into dmin.  fminf ignores a NaN operand, so
// dmin starts as NaN ("no distance seen") and NaN distances are skipped like the reference's `minr >= r`.
__device__ __forceinline__ float dwa_min_d2(float dmin, float px, float py, const float2* ob, int n_ob) {
  for (int j = 0; j < n_ob; ++j) {
    const float dx = px - ob[j].x, dy = py - ob[j].y;
    dmin = fminf(dmin, dx * dx + dy * dy);
  }
  return dmin;
}

// calc_obstacle_cost :77-101 from the smallest squared distance over the checked points.  The reference takes
// sqrtf per pair, returns FLT_MAX at the first r <= robot_radius and otherwise keeps the minimum r.  A correctly
// rounded sqrtf is monotone, so min r = sqrtf(min d2) and "some r <= radius" is "sqrtf(min d2) <= radius": the
// same result with one square root per sample.
__device__ __forceinline__ float dwa_obstacle_cost(float dmin, float robot_radius) {
  float minr = FLT_MAX;
  if (dmin == dmin) {
    const float r = sqrtf(dmin);
    if (r <= robot_radius) return FLT_MAX;
    if (minr >= r) minr = r;
  }
  return (float)(1.0 / (double)minr);  // 1 / FLT_MAX is a float subnormal: no flush to zero anywhere here
}

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
  float x[5];
#pragma unroll
  for (int f = 0; f < 5; ++f) x[f] = xg[(int64_t)f * n + i];
  const float gx = goalg[i], gy = goalg[n + i];
  const float u_prev1 = ug[n + i];

  // calc_dynamic_window :52-60; std::max(a, b) is (a < b) ? b : a and std::min(a, b) is (b < a) ? b : a
  const float lv = x[3] - p.max_accel * p.dt, hv = x[3] + p.max_accel * p.dt;
  const float lw = x[4] - p.max_dyawrate * p.dt, hw = x[4] + p.max_dyawrate * p.dt;
  const float dw0 = (lv < p.min_speed) ? p.min_speed : lv;
  const float dw1 = (p.max_speed < hv) ? p.max_speed : hv;
  const float dw2 = (lw < -p.max_yawrate) ? -p.max_yawrate : lw;
  const float dw3 = (p.max_yawrate < hw) ? p.max_yawrate : hw;
  // the sample grid :126-127: the k-th value is k sequential float adds (every lane runs the sequence, each
  // stores its own entries)
  int nv = 0, nw = 0;
  for (float v = dw0; nv < CRB_DWA_MAX_SPEED_SAMPLES && v <= dw1; v = v + p.v_reso, ++nv)
    if ((nv & 31) == lane) s_v[warp][nv] = v;
  for (float w = dw2; nw < CRB_DWA_MAX_YAWRATE_SAMPLES && w <= dw3; w = w + p.yawrate_reso, ++nw)
    if ((nw & 31) == lane) s_w[warp][nw] = w;
  __syncwarp();

  const float d0 = dwa_min_d2(__int_as_float(0x7fffffff), x[0], x[1], s_ob, n_ob);  // point 0 is x itself
  const float gmag = sqrtf(gx * gx + gy * gy);
  float best_c = 10000.0f;  // min_cost's initial value (:120): a cost above it never wins
  int best_s = -1;
  const int ns = nv * nw;
  for (int s = lane; s < ns; s += 32) {
    const int iv = s / nw;
    const float v = s_v[warp][iv], w = s_w[warp][s - iv * nw];
    float st[5] = {x[0], x[1], x[2], x[3], x[4]};
    float dmin = d0;
    for (int k = 1; k <= n_steps; ++k) {  // calc_trajectory :63-74; obstacles on points 0, 2, 4, ... (:82)
      crb_dwa_motion(st, v, w, p.dt);
      if (!(k & 1)) dmin = dwa_min_d2(dmin, st[0], st[1], s_ob, n_ob);
    }
    // calc_to_goal_cost :103-113: std::pow(float, 2) promotes to double
    const float tmag = (float)sqrt((double)st[0] * (double)st[0] + (double)st[1] * (double)st[1]);
    const float dot = gx * st[0] + gy * st[1];
    const float to_goal = p.to_goal_cost_gain * crb_dwa_acosf(dot / (gmag * tmag));
    const float speed = p.speed_cost_gain * (p.max_speed - st[3]);
    const float cost = to_goal + speed + dwa_obstacle_cost(dmin, p.robot_radius);
    if (cost <= best_c) {  // `min_cost >= final_cost` (:136): within a lane s increases, so ties go to the later
      best_c = cost;
      best_s = s;
    }
  }
  // across lanes: the smaller cost, on a tie the larger index (= the reference's last-wins); NaN never got in
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const float oc = __shfl_xor_sync(0xffffffffu, best_c, off);
    const int os = __shfl_xor_sync(0xffffffffu, best_s, off);
    if (oc < best_c || (oc == best_c && os > best_s)) {
      best_c = oc;
      best_s = os;
    }
  }
  const int biv = best_s >= 0 ? best_s / nw : 0;
  const float bv = best_s >= 0 ? s_v[warp][biv] : 0.0f;
  const float bw = best_s >= 0 ? s_w[warp][best_s - biv * nw] : u_prev1;
  if (lane == 0) {
    ug[i] = bv;
    ug[n + i] = bw;
    if (costg) costg[i] = best_c;
    if (bestg) bestg[i] = best_s;
  }
  if (trajg) {
    if (best_s < 0) {
      for (int f = lane; f < 5 * (n_steps + 1); f += 32) trajg[(int64_t)f * n + i] = __int_as_float(0x7fc00000);
    } else {
      float st[5] = {x[0], x[1], x[2], x[3], x[4]};
      for (int k = 0; k <= n_steps; ++k) {
        if (k > 0) crb_dwa_motion(st, bv, bw, p.dt);
        if ((k & 31) == lane) {
#pragma unroll
          for (int j = 0; j < 5; ++j) trajg[(int64_t)(5 * k + j) * n + i] = st[j];
        }
      }
    }
  }
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

static bool finite_pos(float v) { return isfinite(v) && v > 0.0f; }

// Parameter limits of crb.h; *n_steps = the reference's rollout step count (:67-72), itself bounded.
static int dwa_check_params(const crb_dwa_params* p, int* n_steps) {
  CRB_REQUIRE(p != nullptr, "params is NULL");
  const float* f = &p->max_speed;
  for (int k = 0; k < 12; ++k) CRB_REQUIRE(isfinite(f[k]), "every parameter must be finite");
  CRB_REQUIRE(finite_pos(p->v_reso) && finite_pos(p->yawrate_reso) && finite_pos(p->dt),
              "v_reso, yawrate_reso and dt must be > 0");
  const double wv = fmin(2.0 * p->max_accel * p->dt, (double)p->max_speed - p->min_speed);
  CRB_REQUIRE(wv / p->v_reso + 2.0 <= CRB_DWA_MAX_SPEED_SAMPLES,
              "the speed window allows more than CRB_DWA_MAX_SPEED_SAMPLES samples");
  const double ww = fmin(2.0 * p->max_dyawrate * p->dt, 2.0 * (double)p->max_yawrate);
  CRB_REQUIRE(ww / p->yawrate_reso + 2.0 <= CRB_DWA_MAX_YAWRATE_SAMPLES,
              "the yaw-rate window allows more than CRB_DWA_MAX_YAWRATE_SAMPLES samples");
  float t = 0.0f;
  int k = 0;
  while (k <= CRB_DWA_MAX_STEPS && t <= p->predict_time) {
    t += p->dt;
    ++k;
  }
  CRB_REQUIRE(k <= CRB_DWA_MAX_STEPS, "predict_time / dt allows more than CRB_DWA_MAX_STEPS rollout steps");
  *n_steps = k;
  return CRB_OK;
}

// No device, no computation: the entry points say so after validating their arguments (no CPU fallback).
static int dwa_require_device(const char* fn) {
  int count = 0;
  const cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    cudaGetLastError();
    crb_set_error("%s: no usable CUDA device; libcrb has no CPU fallback", fn);
    return CRB_ERR_NO_DEVICE;
  }
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
  if ((rc = dwa_require_device(__func__)) != CRB_OK) return rc;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  crb_dwa_control_kernel<<<(unsigned)((n + DWA_WARPS - 1) / DWA_WARPS), DWA_BLOCK, 0, ctx->stream>>>(
      n, x, u, goal, ob, n_ob, *prm, n_steps, cost, best, traj);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

int crb_dwa_motion_batched(crb_ctx* ctx, int64_t n, float* x, const float* u, float dt) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(n >= 0 && (n + 255) / 256 <= 0x7fffffff, "n out of range");
  CRB_REQUIRE(n == 0 || (x && u), "x or u is NULL");
  CRB_REQUIRE(finite_pos(dt), "dt must be finite and > 0");
  const int rc = dwa_require_device(__func__);
  if (rc != CRB_OK) return rc;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  crb_dwa_motion_kernel<<<crb_grid_for(n, 256), 256, 0, ctx->stream>>>(n, x, u, dt);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

}  // extern "C"
