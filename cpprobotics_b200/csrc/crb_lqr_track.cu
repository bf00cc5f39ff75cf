// crb_lqr_track.cu — LQR path tracking (lqr_steering_control with calc_nearest_index, and update) for a fleet on
// one course or on a course per vehicle, for sm_90a.
//
// Replaces lqr_steering_control() of src/lqr_steer_control.cpp:98-133 (4 states, 1 input) and
// src/lqr_speed_steer_control.cpp:108-151 (5 states, 2 inputs), each with its calc_nearest_index() (:55-73 /
// :65-83) and solve_DARE() + dlqr(), and update() of both programs (:136-146 / :154-164).  Bit-exact with the
// reference compiled for x86-64: float arithmetic without contraction (-fmad=false, sequential-k sums), the double
// macros DT and L promoting what they touch, YAW_P2P in double (mptg_yaw_p2p), glibc's atan2f for the nearest
// point's bearing (crb_atan2f_libm), glibc's double atan2 narrowed to float for the feed-forward
// (crb_atan2_1_to_float, DESIGN.md §3.4), and update's glibc sinf / cosf / tanf (crb_plant_step).
//
// Mapping: one thread per vehicle, everything in registers.  The course is shared by the fleet, so each block
// streams (cx, cy) through shared memory in tiles and every thread scans each tile in index order: all lanes read
// the same element (a broadcast), and the strict-'<' first minimum holds by construction.  cyaw, ck and sp are read
// once, at the winning index.  Then the DARE iteration of crb_lqr_dare.cuh, which dominates (41-150 iterations of
// 4x4 or 5x5 register algebra).  With a course per vehicle (crb_lqr_track_many_kernel) the vehicles of a block read
// different courses, so each warp searches one vehicle's course at a time with coalesced loads, then every thread
// runs the same per-vehicle body (lqrt_control_vehicle) as the shared-course kernel.
#include <float.h>
#include <math.h>

#include "crb_lqr_dare.cuh"
#include "crb_plant.cuh"

#define LQRT_BLOCK 128
#define LQRT_TILE 2048  // course points per shared-memory tile: (cx, cy) pairs, 16 KB

namespace {

struct LqrtC {
  double dt, wheelbase;
  float Q[25], R[4];
  int maxiter;
  float eps;
};

__device__ __forceinline__ float lqrt_nan() { return __int_as_float(0x7fffffff); }

// A vehicle the reference would read out of bounds for: u and K NaN, iters 0, the status; ind, pe, pth_e untouched.
template <int NX, int NU>
__device__ __forceinline__ void lqrt_refuse(int64_t i, int64_t n, float* __restrict__ u, float* __restrict__ Kg,
                                            int32_t* __restrict__ itg, int32_t* __restrict__ stg, int32_t status) {
  const float q = lqrt_nan();
#pragma unroll
  for (int r = 0; r < NU; ++r) u[(int64_t)r * n + i] = q;
  if (Kg) {
#pragma unroll
    for (int f = 0; f < NX * NU; ++f) Kg[(int64_t)f * n + i] = q;
  }
  if (itg) itg[i] = 0;
  if (stg) stg[i] = status;
}

// lqr_steering_control for vehicle i after calc_nearest_index's scan of its course (cx .. sp, ncourse points): win is
// the first strict minimum (-1 when no point won) and mind its squared distance (FLT_MAX when none won).  The errors,
// A and B, the DARE, -K x, the feed-forward and the stores; both tracking kernels run it.
template <int NX, int NU>
__device__ __forceinline__ void lqrt_control_vehicle(const int64_t i, const int64_t n, const float* __restrict__ state,
                                                     const float sx, const float sy, const float* __restrict__ cx,
                                                     const float* __restrict__ cy, const float* __restrict__ cyaw,
                                                     const float* __restrict__ ck, const float* __restrict__ sp,
                                                     const int ncourse, const LqrtC& c, const int win, const float mind,
                                                     int32_t* __restrict__ ind, float* __restrict__ pe,
                                                     float* __restrict__ pth_e, float* __restrict__ u,
                                                     float* __restrict__ Kg, int32_t* __restrict__ itg,
                                                     int32_t* __restrict__ stg) {
  constexpr int NN = NX * NX, NB = NX * NU;
  // ind is only assigned when a point wins: the 4-state program's persists across calls, the 5-state one's is a
  // local starting at 0 (:110)
  const int j = win >= 0 ? win : (NX == 4 ? ind[i] : 0);
  if (j < 0 || j >= ncourse) {  // the reference reads cx[ind] out of bounds
    lqrt_refuse<NX, NU>(i, n, u, Kg, itg, stg, CRB_LQR_TRACK_BAD_INDEX);
    return;
  }
  const float syaw = state[2 * n + i], sv = state[3 * n + i];
  const float cyaw_j = cyaw[j];
  // :67-72 / :77-82: the error's sign from the course heading against the bearing to the point
  const float angle = mptg_yaw_p2p(cyaw_j - crb_atan2f_libm(cy[j] - sy, cx[j] - sx));
  const float e = angle < 0 ? mind * -1 : mind;

  // lqr_steering_control :101-121 / :111-134
  const float k = ck[j];
  const float th_e = mptg_yaw_p2p(syaw - cyaw_j);
  const double DT = c.dt, L = c.wheelbase;
  float A[NN], B[NB], Q[NN], R[NU * NU], X[NN], K[NB];
#pragma unroll
  for (int f = 0; f < NN; ++f) A[f] = 0.0f;
#pragma unroll
  for (int f = 0; f < NB; ++f) B[f] = 0.0f;
  A[0 + NX * 0] = 1.0f;
  A[0 + NX * 1] = (float)DT;
  A[1 + NX * 2] = sv;
  A[2 + NX * 2] = 1.0f;
  A[2 + NX * 3] = (float)DT;
  B[3] = (float)((double)sv / L);
  if (NX == 5) {
    A[4 + NX * 4] = 1.0f;
    B[4 + NX * 1] = (float)DT;
  }
#pragma unroll
  for (int r = 0; r < NX; ++r)
#pragma unroll
    for (int q = 0; q < NX; ++q) Q[r + NX * q] = c.Q[r + 5 * q];
#pragma unroll
  for (int r = 0; r < NU; ++r)
#pragma unroll
    for (int q = 0; q < NU; ++q) R[r + NU * q] = c.R[r + 2 * q];
  bool converged;
  const int it = crb_lqr_dlqr<NX, NU>(A, B, Q, R, c.maxiter, c.eps, K, X, &converged);

  float x[NX];
  x[0] = e;
  x[1] = (float)((double)(e - pe[i]) / DT);
  x[2] = th_e;
  x[3] = (float)((double)(th_e - pth_e[i]) / DT);
  if (NX == 5) x[NX - 1] = sv - sp[j];
  float us[NU];  // -K * x: the negated gain times x, sequential-k sums
#pragma unroll
  for (int r = 0; r < NU; ++r) {
    float s = (-K[r]) * x[0];
#pragma unroll
    for (int q = 1; q < NX; ++q) s = s + (-K[r + NU * q]) * x[q];
    us[r] = s;
  }
  const float ff = crb_atan2_1_to_float(L * (double)k);
  const float fb = mptg_yaw_p2p(us[0]);
  const float delta = ff + fb;
  if (NU == 1) {
    u[i] = delta;
  } else {
    u[i] = us[NU - 1];  // ai
    u[n + i] = delta;
  }
  ind[i] = j;
  pe[i] = e;
  pth_e[i] = th_e;
  if (Kg) {
#pragma unroll
    for (int f = 0; f < NB; ++f) Kg[(int64_t)f * n + i] = K[f];
  }
  if (itg) itg[i] = it;
  if (stg) stg[i] = converged ? CRB_LQR_TRACK_OK : CRB_LQR_TRACK_DARE_MAXITER;
}

template <int NX, int NU>
__global__ void __launch_bounds__(LQRT_BLOCK)
crb_lqr_steering_control_kernel(int64_t n, const float* __restrict__ state, const float* __restrict__ cx,
                                const float* __restrict__ cy, const float* __restrict__ cyaw,
                                const float* __restrict__ ck, const float* __restrict__ sp, int ncourse,
                                const LqrtC c, int32_t* __restrict__ ind, float* __restrict__ pe,
                                float* __restrict__ pth_e, float* __restrict__ u, float* __restrict__ Kg,
                                int32_t* __restrict__ itg, int32_t* __restrict__ stg) {
  __shared__ float2 tile[LQRT_TILE];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = i < n;
  float sx = 0.0f, sy = 0.0f;
  if (live) { sx = state[i]; sy = state[n + i]; }

  // calc_nearest_index :55-66 / :65-76: the whole course, d_e in float, strict '<' against FLT_MAX
  float mind = FLT_MAX;
  int win = -1;
  for (int base = 0; base < ncourse; base += LQRT_TILE) {
    const int cnt = min(LQRT_TILE, ncourse - base);
    __syncthreads();  // the previous tile is consumed
    for (int j = threadIdx.x; j < cnt; j += LQRT_BLOCK) tile[j] = make_float2(cx[base + j], cy[base + j]);
    __syncthreads();
    if (live) {
      for (int j = 0; j < cnt; ++j) {
        const float2 p = tile[j];
        const float idx = p.x - sx;
        const float idy = p.y - sy;
        const float d_e = idx * idx + idy * idy;
        if (d_e < mind) { mind = d_e; win = base + j; }
      }
    }
  }
  if (!live) return;
  lqrt_control_vehicle<NX, NU>(i, n, state, sx, sy, cx, cy, cyaw, ck, sp, ncourse, c, win, mind, ind, pe, pth_e, u, Kg,
                               itg, stg);
}

// The course [off, off + len) of vehicle i, checked before any course data is read: course_of[i] in [0, n_courses),
// 0 <= course_off[c] < course_off[c + 1] <= npts and a length that fits in int.  len = -1 for a bad reference.
__device__ __forceinline__ void track_course_of(int64_t i, const int64_t* __restrict__ course_off, int32_t n_courses,
                                                int64_t npts, const int32_t* __restrict__ course_of, int64_t& off,
                                                int& len) {
  off = 0;
  len = -1;
  const int32_t c = course_of[i];
  if (c < 0 || c >= n_courses) return;
  const int64_t a = course_off[c], b = course_off[c + 1];
  if (a < 0 || a >= b || b > npts || b - a > 0x7fffffff) return;
  off = a;
  len = (int)(b - a);
}

// lqr_steering_control with a course per vehicle.  Phase 1: each warp searches the courses of its 32 vehicles one at a
// time, the lanes striding the course with coalesced loads, each lane keeping its own strict-'<' first minimum; a
// butterfly argmin on (d_e, index) then gives every lane the winner.  That is the reference's sequential scan: NaN
// never compares less and a distance must be < FLT_MAX to win (a lane without a winner holds (FLT_MAX, INT_MAX),
// which loses to every candidate), the smaller distance wins, and among equal distances the lower index, which is
// the first minimum of the scan in index order.  The lane whose vehicle it is keeps the result in registers.
// Phase 2: one thread per vehicle runs lqrt_control_vehicle on its own course.
template <int NX, int NU>
__global__ void __launch_bounds__(LQRT_BLOCK)
crb_lqr_track_many_kernel(int64_t n, const float* __restrict__ state, const float* __restrict__ cx,
                          const float* __restrict__ cy, const float* __restrict__ cyaw, const float* __restrict__ ck,
                          const float* __restrict__ sp, const int64_t* __restrict__ course_off, int32_t n_courses,
                          int64_t npts, const int32_t* __restrict__ course_of, const LqrtC c,
                          int32_t* __restrict__ ind, float* __restrict__ pe, float* __restrict__ pth_e,
                          float* __restrict__ u, float* __restrict__ Kg, int32_t* __restrict__ itg,
                          int32_t* __restrict__ stg) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const bool live = i < n;
  int64_t off = 0;
  int len = 0;  // 0 for a lane past n: nothing to search
  float sx = 0.0f, sy = 0.0f;
  if (live) {
    track_course_of(i, course_off, n_courses, npts, course_of, off, len);
    if (len > 0) { sx = state[i]; sy = state[n + i]; }
  }

  // calc_nearest_index :55-66 / :65-76 for each vehicle of the warp in turn (k is warp-uniform)
  float mind = FLT_MAX;
  int win = -1;
  for (int k = 0; k < 32; ++k) {
    const int kl = __shfl_sync(0xffffffffu, len, k);
    if (kl <= 0) continue;
    const int64_t ko = __shfl_sync(0xffffffffu, off, k);
    const float kx = __shfl_sync(0xffffffffu, sx, k), ky = __shfl_sync(0xffffffffu, sy, k);
    const float* __restrict__ px = cx + ko;
    const float* __restrict__ py = cy + ko;
    float d = FLT_MAX;
    int w = 0x7fffffff;
    for (int j = lane; j < kl; j += 32) {
      const float idx = px[j] - kx;
      const float idy = py[j] - ky;
      const float d_e = idx * idx + idy * idy;
      if (d_e < d) { d = d_e; w = j; }
    }
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) {
      const float od = __shfl_xor_sync(0xffffffffu, d, s);
      const int ow = __shfl_xor_sync(0xffffffffu, w, s);
      if (od < d || (od == d && ow < w)) { d = od; w = ow; }
    }
    if (lane == k && w != 0x7fffffff) { mind = d; win = w; }
  }
  if (!live) return;
  if (len < 0) {
    lqrt_refuse<NX, NU>(i, n, u, Kg, itg, stg, CRB_LQR_TRACK_BAD_COURSE);
    return;
  }
  lqrt_control_vehicle<NX, NU>(i, n, state, sx, sy, cx + off, cy + off, cyaw + off, ck + off, sp ? sp + off : nullptr,
                               len, c, win, mind, ind, pe, pth_e, u, Kg, itg, stg);
}

__global__ void __launch_bounds__(256)
crb_lqr_update_kernel(int64_t n, float* __restrict__ state, const float* __restrict__ a,
                      const float* __restrict__ delta, const PlantC k) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float x = state[i], y = state[n + i], yaw = state[2 * n + i], v = state[3 * n + i];
  crb_plant_step(x, y, yaw, v, a[i], delta[i], k);
  state[i] = x; state[n + i] = y; state[2 * n + i] = yaw; state[3 * n + i] = v;
}

int lqrt_check_plant(const crb_lqr_track_params* p) {
  CRB_REQUIRE(p != nullptr, "prm is NULL");
  CRB_REQUIRE(isfinite(p->dt) && isfinite(p->wheelbase), "dt and wheelbase must be finite");
  CRB_REQUIRE(isfinite(p->max_steer) && fabs(p->max_steer) < 120.0, "max_steer must be finite with |max_steer| < 120");
  return CRB_OK;
}

// The host checks both control entry points share: nx, n, sp against nx, and the parameters.
int lqrt_check_control(int nx, int64_t n, const float* sp, const crb_lqr_track_params* prm) {
  CRB_REQUIRE(nx == 4 || nx == 5, "nx must be 4 (lqr_steer_control) or 5 (lqr_speed_steer_control)");
  CRB_REQUIRE(n >= 0 && (n + LQRT_BLOCK - 1) / LQRT_BLOCK <= 0x7fffffff, "n out of range");
  CRB_REQUIRE((sp != nullptr) == (nx == 5), "sp must be given for nx = 5 and NULL for nx = 4");
  const int rc = lqrt_check_plant(prm);
  if (rc) return rc;
  for (int f = 0; f < 25; ++f) CRB_REQUIRE(isfinite(prm->Q[f]), "Q must be finite");
  for (int f = 0; f < 4; ++f) CRB_REQUIRE(isfinite(prm->R[f]), "R must be finite");
  CRB_REQUIRE(isfinite(prm->eps) && prm->maxiter >= 0, "eps must be finite and maxiter >= 0");
  return CRB_OK;
}

LqrtC lqrt_constants(const crb_lqr_track_params* prm) {
  LqrtC c;
  c.dt = prm->dt;
  c.wheelbase = prm->wheelbase;
  for (int f = 0; f < 25; ++f) c.Q[f] = prm->Q[f];
  for (int f = 0; f < 4; ++f) c.R[f] = prm->R[f];
  c.maxiter = prm->maxiter;
  c.eps = prm->eps;
  return c;
}

}  // namespace

extern "C" {

void crb_lqr_track_default_params(crb_lqr_track_params* p, int nx) {
  // src/lqr_steer_control.cpp:20-23 / src/lqr_speed_steer_control.cpp:20-23 (DT, L, MAX_STEER), :77-78 / :87-88
  // (maxiter, eps), :114-115 / :131-132 (Q, R)
  p->dt = 0.1;
  p->wheelbase = 0.5;
  p->max_steer = 45.0 / 180 * 3.14159265358979323846;
  for (int f = 0; f < 25; ++f) p->Q[f] = (f % 6 == 0) ? 1.0f : 0.0f;
  for (int f = 0; f < 4; ++f) p->R[f] = 0.0f;
  p->R[0] = 1.0f;
  if (nx != 4) p->R[3] = 1.0f;
  p->maxiter = 150;
  p->eps = (float)0.01;
}

int crb_lqr_steering_control_batched(crb_ctx* ctx, int64_t n, int nx, const float* state, const float* cx,
                                     const float* cy, const float* cyaw, const float* ck, const float* sp,
                                     int32_t ncourse, const crb_lqr_track_params* prm, int32_t* ind, float* pe,
                                     float* pth_e, float* u, float* K, int32_t* iters, int32_t* status) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(ncourse >= 1, "ncourse must be >= 1");
  const int rc = lqrt_check_control(nx, n, sp, prm);
  if (rc) return rc;
  CRB_REQUIRE(n == 0 || (state && cx && cy && cyaw && ck && ind && pe && pth_e && u), "NULL array");
  const int dev = crb_require_device(__func__);
  if (dev) return dev;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);   // ctx->device is current for this call, the caller's device is restored after it
  const LqrtC c = lqrt_constants(prm);
  const int grid = crb_grid_for(n, LQRT_BLOCK);
  if (nx == 4)
    crb_lqr_steering_control_kernel<4, 1><<<grid, LQRT_BLOCK, 0, ctx->stream>>>(
        n, state, cx, cy, cyaw, ck, sp, ncourse, c, ind, pe, pth_e, u, K, iters, status);
  else
    crb_lqr_steering_control_kernel<5, 2><<<grid, LQRT_BLOCK, 0, ctx->stream>>>(
        n, state, cx, cy, cyaw, ck, sp, ncourse, c, ind, pe, pth_e, u, K, iters, status);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

int crb_lqr_steering_control_many_batched(crb_ctx* ctx, int64_t n, int nx, const float* state, const float* cx,
                                          const float* cy, const float* cyaw, const float* ck, const float* sp,
                                          const int64_t* course_off, int32_t n_courses, int64_t npts,
                                          const int32_t* course_of, const crb_lqr_track_params* prm, int32_t* ind,
                                          float* pe, float* pth_e, float* u, float* K, int32_t* iters,
                                          int32_t* status) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(n_courses >= 1 && npts >= 1, "n_courses and npts must be >= 1");
  const int rc = lqrt_check_control(nx, n, sp, prm);
  if (rc) return rc;
  CRB_REQUIRE(n == 0 || (state && cx && cy && cyaw && ck && course_off && course_of && ind && pe && pth_e && u),
              "NULL array");
  const int dev = crb_require_device(__func__);
  if (dev) return dev;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  const LqrtC c = lqrt_constants(prm);
  const int grid = crb_grid_for(n, LQRT_BLOCK);
  if (nx == 4)
    crb_lqr_track_many_kernel<4, 1><<<grid, LQRT_BLOCK, 0, ctx->stream>>>(
        n, state, cx, cy, cyaw, ck, sp, course_off, n_courses, npts, course_of, c, ind, pe, pth_e, u, K, iters, status);
  else
    crb_lqr_track_many_kernel<5, 2><<<grid, LQRT_BLOCK, 0, ctx->stream>>>(
        n, state, cx, cy, cyaw, ck, sp, course_off, n_courses, npts, course_of, c, ind, pe, pth_e, u, K, iters, status);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

int crb_lqr_update_batched(crb_ctx* ctx, int64_t n, float* state, const float* a, const float* delta,
                           const crb_lqr_track_params* prm) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(n >= 0 && (n + 255) / 256 <= 0x7fffffff, "n out of range");
  const int rc = lqrt_check_plant(prm);
  if (rc) return rc;
  CRB_REQUIRE(n == 0 || (state && a && delta), "NULL array");
  const int dev = crb_require_device(__func__);
  if (dev) return dev;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  PlantC k;
  k.max_steer = prm->max_steer;
  k.dt = prm->dt;
  k.wb = prm->wheelbase;
  k.max_speed = HUGE_VAL;   // the LQR programs' update has no speed clamp
  k.min_speed = -HUGE_VAL;
  crb_lqr_update_kernel<<<crb_grid_for(n, 256), 256, 0, ctx->stream>>>(n, state, a, delta, k);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

}  // extern "C"
