// crb_mptg.cu — model-predictive trajectory generation (TrajectoryOptimizer::optimizer_traj) for a batch of
// problems, for sm_90a.
//
// Replaces optimizer_traj() of include/trajectory_optimizer.h:53-200 and MotionModel::generate_trajectory /
// generate_last_state of include/motion_model.h:59-150 for n independent (start, target, initial parameter)
// problems.  Bit-exact with the reference compiled for x86-64: every float operation separately rounded (explicit
// __f*_rn / __d*_rn intrinsics, so the TU's -fmad setting does not matter), YAW_P2P and the cost's std::pow /
// std::sqrt in double, Eigen 3.3's 3x3 cofactor inverse, glibc's sinf / cosf (crb_sincosf_libm) and tanf
// (crb_tanf_libm), and the reference's own float accumulation of the roll-out's time variable.
//
// Mapping: one thread per problem, all state in registers.  An iteration rolls out the 6 Jacobian parameters in
// lockstep (their step counts differ by a few steps at most; finished ones are masked), then the 2 line-search
// candidates together.  Two savings that keep the bits: the next iteration's nominal roll-out is the chosen
// line-search candidate (`p.distance += alpha * dp(0)` is the same expression as the candidate's), so it is not
// rolled out again; and the returned trajectory is regenerated once at exit from the saved parameter instead of
// being stored every iteration.
#include <float.h>

#include "crb_common.cuh"

#define MPTG_BLOCK 128

namespace {

constexpr double kPi = 3.14159265358979323846;  // M_PI
constexpr double kTwoPi = 2.0 * kPi;             // 2*M_PI (an exact doubling)

// fmod(a, 2*M_PI), exactly.  fmod is exact in IEEE arithmetic; for |a| < 4 pi (every wrapped yaw) its result is
// a itself or a -+ 2 pi, and that subtraction is exact (Sterbenz), so the general routine is only needed beyond.
__device__ __forceinline__ double mptg_fmod_2pi(double a) {
  const double aa = fabs(a);
  if (aa < kTwoPi) return a;
  if (aa < 2.0 * kTwoPi) return copysign(__dsub_rn(aa, kTwoPi), a);  // fmod's result has a's sign
  return fmod(a, kTwoPi);
}

// YAW_P2P(angle) :18 on a float, in double, narrowed back to float by the assignment
__device__ __forceinline__ float mptg_yaw_p2p(float yaw) {
  double a = mptg_fmod_2pi(__dadd_rn((double)yaw, kPi));
  a = mptg_fmod_2pi(__dsub_rn(a, kTwoPi));
  return __double2float_rn(__dadd_rn(a, kPi));
}

// Eigen 3.3 compute_inverse<Matrix3f, Matrix3f, 3>: cofactor_3x3<i,j> = m(i1,j1) m(i2,j2) - m(i1,j2) m(i2,j1)
// with i1 = (i+1)%3, i2 = (i+2)%3 (likewise j); det = (c00 m00 + c10 m10) + c20 m20; out(i,j) =
// cofactor_3x3<j,i> * (1 / det).  m[r][c].
__device__ __forceinline__ float mptg_cof(const float (&m)[3][3], int i, int j) {
  const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
  return __fsub_rn(__fmul_rn(m[i1][j1], m[i2][j2]), __fmul_rn(m[i1][j2], m[i2][j1]));
}
// out = inverse(m) * y, the product summed in k order
__device__ __forceinline__ void mptg_inv_mul(const float (&m)[3][3], const float (&y)[3], float (&out)[3]) {
  const float c0 = mptg_cof(m, 0, 0), c1 = mptg_cof(m, 1, 0), c2 = mptg_cof(m, 2, 0);
  const float det = __fadd_rn(__fadd_rn(__fmul_rn(c0, m[0][0]), __fmul_rn(c1, m[1][0])), __fmul_rn(c2, m[2][0]));
  const float invdet = __fdiv_rn(1.0f, det);
  float inv[3][3];
  inv[0][0] = __fmul_rn(c0, invdet);
  inv[0][1] = __fmul_rn(c1, invdet);
  inv[0][2] = __fmul_rn(c2, invdet);
#pragma unroll
  for (int i = 1; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) inv[i][j] = __fmul_rn(mptg_cof(m, j, i), invdet);
#pragma unroll
  for (int i = 0; i < 3; ++i)
    out[i] = __fadd_rn(__fadd_rn(__fmul_rn(inv[i][0], y[0]), __fmul_rn(inv[i][1], y[1])), __fmul_rn(inv[i][2], y[2]));
}

// One roll-out of generate_last_state / generate_trajectory in progress.
struct Roll {
  float x, y, yaw, t, horizon, dt, c0, c1, c2;
  int steps;
};

// :111-122: n = distance / ds, horizon = distance / v, the steering polynomial from quadratic_interpolation
// ({0, horizon/2, horizon}, steering) :59-72 (std::pow(float, 2) is an exact double square: a rounded float product)
__device__ __forceinline__ void mptg_setup(Roll& r, const float (&st)[4], float ds, float d, float s0, float s1,
                                           float s2) {
  const float n = __fdiv_rn(d, ds);
  r.horizon = __fdiv_rn(d, st[3]);
  r.dt = __fdiv_rn(r.horizon, n);
  const float h2 = __fdiv_rn(r.horizon, 2.0f);
  const float A[3][3] = {{__fmul_rn(0.0f, 0.0f), 0.0f, 1.0f},
                         {__fmul_rn(h2, h2), h2, 1.0f},
                         {__fmul_rn(r.horizon, r.horizon), r.horizon, 1.0f}};
  const float Y[3] = {s0, s1, s2};
  float c[3];
  mptg_inv_mul(A, Y, c);
  r.c0 = c[0];
  r.c1 = c[1];
  r.c2 = c[2];
  r.x = st[0];
  r.y = st[1];
  r.yaw = st[2];
  r.t = 0.0f;
  r.steps = 0;
}

// One pass of the loop body :125-128 / :146-147 (MotionModel::update :102-108); false when kp is outside
// crb_tanf_libm's proven range (nothing is changed then).
__device__ __forceinline__ bool mptg_step(Roll& r, float v, float v_over_l) {
  const float kp = __fadd_rn(__fadd_rn(__fmul_rn(__fmul_rn(r.c0, r.t), r.t), __fmul_rn(r.c1, r.t)), r.c2);
  if (!crb_tanf_libm_in_range(kp)) return false;
  float sn, cs;
  crb_sincosf_libm(r.yaw, sn, cs);
  const float tn = crb_tanf_libm(kp);
  r.x = __fadd_rn(r.x, __fmul_rn(__fmul_rn(v, cs), r.dt));
  r.y = __fadd_rn(r.y, __fmul_rn(__fmul_rn(v, sn), r.dt));
  r.yaw = mptg_yaw_p2p(__fadd_rn(r.yaw, __fmul_rn(__fmul_rn(v_over_l, tn), r.dt)));
  r.t = __fadd_rn(r.t, r.dt);
  ++r.steps;
  return true;
}

// Runs K set-up roll-outs to their end in lockstep.  Returns 0, or the status that stops the problem:
// CRB_MPTG_OUT_OF_RANGE if any roll-out meets a steering outside the tanf range, else CRB_MPTG_STEP_CAP if any
// needs more than CRB_MPTG_MAX_STEPS steps (the same answer whatever order the roll-outs run in).
template <int K>
__device__ __forceinline__ int mptg_run(Roll (&r)[K], float v, float v_over_l) {
  unsigned live = 0;
#pragma unroll
  for (int k = 0; k < K; ++k)
    if (r[k].t < r[k].horizon) live |= 1u << k;
  bool cap = false;
  while (live) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      if (!((live >> k) & 1u)) continue;
      if (r[k].steps == CRB_MPTG_MAX_STEPS) {
        cap = true;
        live &= ~(1u << k);
        continue;
      }
      if (!mptg_step(r[k], v, v_over_l)) return CRB_MPTG_OUT_OF_RANGE;
      if (!(r[k].t < r[k].horizon)) live &= ~(1u << k);
    }
  }
  return cap ? CRB_MPTG_STEP_CAP : 0;
}

// A roll-out known to complete, writing its first max_pts points to traj (field 3k+j).
__device__ void mptg_write(const float (&st)[4], const crb_mptg_params& p, const float (&q)[4], int max_pts,
                           int64_t n, int64_t i, float* __restrict__ traj) {
  Roll r;
  mptg_setup(r, st, p.ds, q[0], q[1], q[2], q[3]);
  const float vl = __fdiv_rn(st[3], p.base_l);
  while (r.t < r.horizon && r.steps < max_pts) {
    const int k = r.steps;
    mptg_step(r, st[3], vl);
    traj[(3 * (int64_t)k) * n + i] = r.x;
    traj[(3 * (int64_t)k + 1) * n + i] = r.y;
    traj[(3 * (int64_t)k + 2) * n + i] = r.yaw;
  }
}

// calc_diff :130-135 and the cost :108-109
__device__ __forceinline__ float mptg_error(const float (&tg)[3], const Roll& r, float (&e)[3]) {
  e[0] = __fsub_rn(tg[0], r.x);
  e[1] = __fsub_rn(tg[1], r.y);
  e[2] = mptg_yaw_p2p(__fsub_rn(tg[2], r.yaw));
  const double a = __dmul_rn((double)e[0], (double)e[0]), b = __dmul_rn((double)e[1], (double)e[1]),
               c = __dmul_rn((double)e[2], (double)e[2]);
  return __double2float_rn(__dsqrt_rn(__dadd_rn(__dadd_rn(a, b), c)));
}

__device__ __forceinline__ bool mptg_yaw_in_range(float yaw) { return fabsf(yaw) < 120.0f; }

}  // namespace

__global__ void __launch_bounds__(MPTG_BLOCK)
crb_mptg_optimize_kernel(int64_t n, const float* __restrict__ stg, const float* __restrict__ tgg,
                         float* __restrict__ pg, crb_mptg_params prm, int max_pts, float* __restrict__ trajg,
                         int32_t* __restrict__ lenp, float* __restrict__ costp, int32_t* __restrict__ statusp,
                         int32_t* __restrict__ itersp) {
  const int64_t i = (int64_t)blockIdx.x * MPTG_BLOCK + threadIdx.x;
  if (i >= n) return;
  float st[4], tg[3], q[4];
#pragma unroll
  for (int f = 0; f < 4; ++f) st[f] = stg[(int64_t)f * n + i];
#pragma unroll
  for (int f = 0; f < 3; ++f) tg[f] = tgg[(int64_t)f * n + i];
#pragma unroll
  for (int f = 0; f < 4; ++f) q[f] = pg[(int64_t)f * n + i];
  const float v = st[3], vl = __fdiv_rn(v, prm.base_l);
  float h2[3];  // (float)(2.0 * h[k]) :154, :162, :170
#pragma unroll
  for (int k = 0; k < 3; ++k) h2[k] = __double2float_rn(__dmul_rn(2.0, (double)prm.h_step[k]));

  int status = CRB_MPTG_MAX_ITER_REACHED, count = 0;
  int traj_steps = 0;
  float traj_cost = __int_as_float(0x7fc00000);
  float traj_q[4] = {q[0], q[1], q[2], q[3]};
  // the nominal roll-out of the current iteration: its steps, error vector and cost
  int nom_steps = 0;
  float nom_e[3], nom_cost = 0.0f;
  if (!mptg_yaw_in_range(st[2])) {
    status = CRB_MPTG_OUT_OF_RANGE;
  } else if (prm.max_iter > 0) {
    Roll r[1];
    mptg_setup(r[0], st, prm.ds, q[0], q[1], q[2], q[3]);
    const int s = mptg_run(r, v, vl);
    if (s) status = s;
    nom_steps = r[0].steps;
    nom_cost = mptg_error(tg, r[0], nom_e);
  }
  for (int it = 0; status == CRB_MPTG_MAX_ITER_REACHED && it < prm.max_iter; ++it) {
    if (nom_steps == 0) {  // sample_traj.back() of an empty Traj
      status = CRB_MPTG_EMPTY_TRAJ;
      break;
    }
    traj_steps = nom_steps;
    traj_cost = nom_cost;
#pragma unroll
    for (int f = 0; f < 4; ++f) traj_q[f] = q[f];
    if (nom_cost < prm.cost_th) {
      status = CRB_MPTG_CONVERGED;
      break;
    }
    // calc_J :146-175: distance +- h0, steering[1] +- h1, steering[2] +- h2
    Roll r[6];
    mptg_setup(r[0], st, prm.ds, __fadd_rn(q[0], prm.h_step[0]), q[1], q[2], q[3]);
    mptg_setup(r[1], st, prm.ds, __fsub_rn(q[0], prm.h_step[0]), q[1], q[2], q[3]);
    mptg_setup(r[2], st, prm.ds, q[0], q[1], __fadd_rn(q[2], prm.h_step[1]), q[3]);
    mptg_setup(r[3], st, prm.ds, q[0], q[1], __fsub_rn(q[2], prm.h_step[1]), q[3]);
    mptg_setup(r[4], st, prm.ds, q[0], q[1], q[2], __fadd_rn(q[3], prm.h_step[2]));
    mptg_setup(r[5], st, prm.ds, q[0], q[1], q[2], __fsub_rn(q[3], prm.h_step[2]));
    int s = mptg_run(r, v, vl);
    if (s) {
      status = s;
      break;
    }
    float J[3][3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float ep[3], em[3];
      mptg_error(tg, r[2 * c], ep);
      mptg_error(tg, r[2 * c + 1], em);
#pragma unroll
      for (int k = 0; k < 3; ++k) J[k][c] = __fdiv_rn(__fsub_rn(ep[k], em[k]), h2[c]);
    }
    float dp[3];
    mptg_inv_mul(J, nom_e, dp);
#pragma unroll
    for (int k = 0; k < 3; ++k) dp[k] = -dp[k];  // dp = -(J^-1 dc): the sign is exact
    // selection_learning_param :178-200: a = 1.0, 1.5
    Roll ls[2];
    float cq[2][3];
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const float al = a ? 1.5f : 1.0f;
      cq[a][0] = __fadd_rn(q[0], __fmul_rn(al, dp[0]));
      cq[a][1] = __fadd_rn(q[2], __fmul_rn(al, dp[1]));
      cq[a][2] = __fadd_rn(q[3], __fmul_rn(al, dp[2]));
      mptg_setup(ls[a], st, prm.ds, cq[a][0], q[1], cq[a][1], cq[a][2]);
    }
    s = mptg_run(ls, v, vl);
    if (s) {
      status = s;
      break;
    }
    float e1[3], e2[3];
    const float c1 = mptg_error(tg, ls[0], e1), c2 = mptg_error(tg, ls[1], e2);
    float mincost = FLT_MAX;
    int pick = 0;
    if (c1 <= mincost) mincost = c1;
    if (c2 <= mincost) pick = 1;  // the later a wins a tie; a NaN or +inf cost never wins
    q[0] = cq[pick][0];
    q[2] = cq[pick][1];
    q[3] = cq[pick][2];
    ++count;
    nom_steps = pick ? ls[1].steps : ls[0].steps;
    nom_cost = pick ? c2 : c1;
#pragma unroll
    for (int k = 0; k < 3; ++k) nom_e[k] = pick ? e2[k] : e1[k];
  }

  const bool has_traj = status == CRB_MPTG_CONVERGED || status == CRB_MPTG_MAX_ITER_REACHED;
  if (!has_traj) {
    traj_steps = 0;
    traj_cost = __int_as_float(0x7fc00000);
  }
#pragma unroll
  for (int f = 0; f < 4; ++f) pg[(int64_t)f * n + i] = q[f];
  if (lenp) lenp[i] = traj_steps;
  if (costp) costp[i] = traj_cost;
  if (statusp) statusp[i] = status;
  if (itersp) itersp[i] = count;
  if (trajg && traj_steps > 0 && max_pts > 0) mptg_write(st, prm, traj_q, max_pts, n, i, trajg);
}

__global__ void __launch_bounds__(MPTG_BLOCK)
crb_mptg_generate_kernel(int64_t n, const float* __restrict__ stg, const float* __restrict__ pg,
                         crb_mptg_params prm, int max_pts, float* __restrict__ trajg, int32_t* __restrict__ lenp,
                         float* __restrict__ lastg, int32_t* __restrict__ statusp) {
  const int64_t i = (int64_t)blockIdx.x * MPTG_BLOCK + threadIdx.x;
  if (i >= n) return;
  float st[4], q[4];
#pragma unroll
  for (int f = 0; f < 4; ++f) st[f] = stg[(int64_t)f * n + i];
#pragma unroll
  for (int f = 0; f < 4; ++f) q[f] = pg[(int64_t)f * n + i];
  int status = CRB_MPTG_OUT_OF_RANGE;
  Roll r[1];
  if (mptg_yaw_in_range(st[2])) {
    mptg_setup(r[0], st, prm.ds, q[0], q[1], q[2], q[3]);
    status = mptg_run(r, st[3], __fdiv_rn(st[3], prm.base_l));
  }
  const bool ok = status == CRB_MPTG_CONVERGED;
  const float nan = __int_as_float(0x7fc00000);
  if (lenp) lenp[i] = ok ? r[0].steps : 0;
  if (statusp) statusp[i] = status;
  if (lastg) {
    lastg[i] = ok ? r[0].x : nan;
    lastg[n + i] = ok ? r[0].y : nan;
    lastg[2 * n + i] = ok ? r[0].yaw : nan;
  }
  if (trajg && ok && r[0].steps > 0 && max_pts > 0) mptg_write(st, prm, q, max_pts, n, i, trajg);
}

// Parameter limits of crb.h.
static int mptg_check_params(const crb_mptg_params* p, int max_pts) {
  CRB_REQUIRE(p != nullptr, "params is NULL");
  CRB_REQUIRE(isfinite(p->base_l) && isfinite(p->ds) && isfinite(p->cost_th) && isfinite(p->h_step[0]) &&
                  isfinite(p->h_step[1]) && isfinite(p->h_step[2]),
              "every parameter must be finite");
  CRB_REQUIRE(p->ds > 0.0f, "ds must be > 0");
  CRB_REQUIRE(p->base_l != 0.0f, "base_l must be != 0");
  CRB_REQUIRE(p->h_step[0] > 0.0f && p->h_step[1] > 0.0f && p->h_step[2] > 0.0f, "h_step must be > 0");
  CRB_REQUIRE(p->max_iter >= 0 && p->max_iter <= CRB_MPTG_MAX_ITER, "max_iter must be in [0, CRB_MPTG_MAX_ITER]");
  CRB_REQUIRE(max_pts >= 0, "max_pts must be >= 0");
  return CRB_OK;
}

// No device, no computation: the entry points say so after validating their arguments (no CPU fallback).
static int mptg_require_device(const char* fn) {
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

void crb_mptg_default_params(crb_mptg_params* p) {
  // src/model_predictive_trajectory_generator.cpp:19-20 (L, DS), :31-33 (cost_th_, h_step_, max_iter)
  p->base_l = (float)1.0;
  p->ds = (float)0.1;
  p->max_iter = 100;
  p->cost_th = (float)0.1;
  p->h_step[0] = (float)0.2;
  p->h_step[1] = (float)0.005;
  p->h_step[2] = (float)0.005;
}

int crb_mptg_optimize_batched(crb_ctx* ctx, int64_t n, const float* state, const float* target, float* param,
                              const crb_mptg_params* prm, int max_pts, float* traj, int32_t* traj_len,
                              float* cost, int32_t* status, int32_t* iters) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(n >= 0 && (n + MPTG_BLOCK - 1) / MPTG_BLOCK <= 0x7fffffff, "n out of range");
  CRB_REQUIRE(n == 0 || (state && target && param), "state, target or param is NULL");
  int rc = mptg_check_params(prm, max_pts);
  if (rc != CRB_OK) return rc;
  if ((rc = mptg_require_device(__func__)) != CRB_OK) return rc;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  crb_mptg_optimize_kernel<<<crb_grid_for(n, MPTG_BLOCK), MPTG_BLOCK, 0, ctx->stream>>>(
      n, state, target, param, *prm, max_pts, traj, traj_len, cost, status, iters);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

int crb_mptg_generate_trajectory_batched(crb_ctx* ctx, int64_t n, const float* state, const float* param,
                                         const crb_mptg_params* prm, int max_pts, float* traj,
                                         int32_t* traj_len, float* last, int32_t* status) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(n >= 0 && (n + MPTG_BLOCK - 1) / MPTG_BLOCK <= 0x7fffffff, "n out of range");
  CRB_REQUIRE(n == 0 || (state && param), "state or param is NULL");
  int rc = mptg_check_params(prm, max_pts);
  if (rc != CRB_OK) return rc;
  if ((rc = mptg_require_device(__func__)) != CRB_OK) return rc;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  crb_mptg_generate_kernel<<<crb_grid_for(n, MPTG_BLOCK), MPTG_BLOCK, 0, ctx->stream>>>(
      n, state, param, *prm, max_pts, traj, traj_len, last, status);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

}  // extern "C"
