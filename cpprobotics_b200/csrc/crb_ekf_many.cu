// crb_ekf_many.cu — the batched EKF step with a noise model per agent, for sm_90a.
//
// Replaces ekf_estimation(xEst, PEst, z, u, Q, R) of the reference, src/extended_kalman_filter.cpp:64-78, which takes
// Q and R per call, for n agents that each name their model (dt, Q, R) in a device table.  Agent i runs crb_ekf.cu's
// ekf_step (crb_ekf_common.cuh) with models[model_of[i]], so its x and P are bitwise those of crb_ekf_step_batched
// run with that model.
//
// Mapping, launch shapes, PDL and 64-bit offsets are crb_ekf.cu's (one thread per agent or per agent pair).  The
// model record is read through the read-only path right before the step that uses it: agents of one warp mostly
// name different models, so a per-lane load is the general access, and with few models the records stay in L1
// (a one-model table is one broadcast line).  The 88 bytes of a record are eleven 8-byte loads; the record is only
// live across one ekf_step, so the two-agent form holds one record at a time (DESIGN.md §3 has the measurements).
#include <stdint.h>

#include "crb_ekf_common.cuh"

// The record of model m; m must lie in [0, n_models).
__device__ __forceinline__ EkfArgs ekf_model(const EkfArgs* __restrict__ models, int32_t m) {
  const double* r = reinterpret_cast<const double*>(models + m);
  EkfArgs a;
  a.dt = __ldg(r);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float2 q = __ldg(reinterpret_cast<const float2*>(r + 1 + k));
    a.Q[2 * k] = q.x;
    a.Q[2 * k + 1] = q.y;
  }
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const float2 q = __ldg(reinterpret_cast<const float2*>(r + 9 + k));
    a.R[2 * k] = q.x;
    a.R[2 * k + 1] = q.y;
  }
  return a;
}

// crb_ekf_step_kernel with the constants of agent i taken from models[model_of[i]].  An index outside
// [0, n_models) reads no record (model 0 stands in for the arithmetic) and makes the agent's x and P NaN.
template <int BLOCK, int MINB, int V>
__global__ void __launch_bounds__(BLOCK, MINB)
crb_ekf_many_kernel(int64_t count, int64_t ld, float* __restrict__ x, float* __restrict__ P,
                    const float* __restrict__ z, const float* __restrict__ u, int64_t ld_zu, int n_steps,
                    const EkfArgs* __restrict__ models, int32_t n_models, const int32_t* __restrict__ model_of,
                    int32_t* __restrict__ status) {
  const int64_t i = V * ((int64_t)blockIdx.x * blockDim.x + threadIdx.x);
  if (i >= count) return;
  crb_pdl_launch_dependents();   // the next launch may start scheduling its CTAs behind ours
  crb_pdl_wait();   // the previous launch on this stream (e.g. the preceding filter step) is complete
  int32_t m[V];
  if constexpr (V == 1) {
    m[0] = __ldcs(model_of + i);
  } else {
    const int2 t = __ldcs(reinterpret_cast<const int2*>(model_of + i));
    m[0] = t.x;
    m[1] = t.y;
  }
  bool ok[V];
#pragma unroll
  for (int k = 0; k < V; ++k) {
    ok[k] = (uint32_t)m[k] < (uint32_t)n_models;
    if (!ok[k]) m[k] = 0;
  }
  float xs[4][V], Ps[16][V], z0[V], z1[V], u0[V], u1[V];
#pragma unroll
  for (int f = 0; f < 4; ++f) ld_agents<V>(x + f * ld + i, xs[f]);
#pragma unroll
  for (int f = 0; f < 16; ++f) ld_agents<V>(P + f * ld + i, Ps[f]);
  ld_agents<V>(z + 0 * ld_zu + i, z0);
  ld_agents<V>(z + 1 * ld_zu + i, z1);
  ld_agents<V>(u + 0 * ld_zu + i, u0);
  ld_agents<V>(u + 1 * ld_zu + i, u1);
  for (int s = 0; s < n_steps; ++s) {
    float nz0[V] = {}, nz1[V] = {}, nu0[V] = {}, nu1[V] = {};
    if (s + 1 < n_steps) {  // prefetch the next step's observation/control under this step's math
      const int64_t o = (int64_t)(s + 1) * 2;
      ld_agents<V>(z + (o + 0) * ld_zu + i, nz0);
      ld_agents<V>(z + (o + 1) * ld_zu + i, nz1);
      ld_agents<V>(u + (o + 0) * ld_zu + i, nu0);
      ld_agents<V>(u + (o + 1) * ld_zu + i, nu1);
    }
#pragma unroll
    for (int k = 0; k < V; ++k) {
      float xk[4], Pk[16];
#pragma unroll
      for (int f = 0; f < 4; ++f) xk[f] = xs[f][k];
#pragma unroll
      for (int f = 0; f < 16; ++f) Pk[f] = Ps[f][k];
      const EkfArgs a = ekf_model(models, m[k]);
      ekf_step(xk, Pk, z0[k], z1[k], u0[k], u1[k], a);
#pragma unroll
      for (int f = 0; f < 4; ++f) xs[f][k] = xk[f];
#pragma unroll
      for (int f = 0; f < 16; ++f) Ps[f][k] = Pk[f];
      z0[k] = nz0[k]; z1[k] = nz1[k]; u0[k] = nu0[k]; u1[k] = nu1[k];
    }
  }
  const float nan = __int_as_float(0x7fffffff);
#pragma unroll
  for (int k = 0; k < V; ++k) {
    if (!ok[k]) {  // a filter whose step did not run must not look as if it had
#pragma unroll
      for (int f = 0; f < 4; ++f) xs[f][k] = nan;
#pragma unroll
      for (int f = 0; f < 16; ++f) Ps[f][k] = nan;
    }
    if (status) status[i + k] = ok[k] ? CRB_EKF_OK : CRB_EKF_BAD_MODEL;
  }
  // store addresses recomputed after the math, as in crb_ekf_step_kernel (which says why)
  int64_t lds = ld, is = i;
  asm volatile("" : "+l"(lds), "+l"(is));
#pragma unroll
  for (int f = 0; f < 4; ++f) st_agents<V>(x + f * lds + is, xs[f]);
#pragma unroll
  for (int f = 0; f < 16; ++f) st_agents<V>(P + f * lds + is, Ps[f]);
}

int ekf_many_launch(crb_ctx* ctx, cudaStream_t st, int64_t count, int64_t ld, float* x, float* P, const float* z,
                    const float* u, int64_t ld_zu, int n_steps, const crb_ekf_params* models, int32_t n_models,
                    const int32_t* model_of, int32_t* status) {
  const EkfArgs* tab = reinterpret_cast<const EkfArgs*>(models);
  // crb_ekf.cu's ekf_launch selection, with model_of read 8 bytes at a time in the two-agent form
  const bool pair_ok = (count % 2) == 0 && (ld % 2) == 0 && (ld_zu % 2) == 0 &&
                       (((uintptr_t)x | (uintptr_t)P | (uintptr_t)z | (uintptr_t)u | (uintptr_t)model_of) & 7) == 0;
  if (pair_ok)
    CRB_CUDA(crb_launch_pdl(crb_ekf_many_kernel<128, 4, 2>, (unsigned)crb_grid_for(count / 2, 128), 128u, st,
                            count, ld, x, P, z, u, ld_zu, n_steps, tab, n_models, model_of, status));
  else
    CRB_CUDA(crb_launch_pdl(crb_ekf_many_kernel<256, 3, 1>, (unsigned)crb_grid_for(count, 256), 256u, st,
                            count, ld, x, P, z, u, ld_zu, n_steps, tab, n_models, model_of, status));
  ctx->launches++;
  return CRB_OK;
}

extern "C" int crb_ekf_step_many_batched(crb_ctx* ctx, int64_t n, float* x, float* P, const float* z, const float* u,
                                         const crb_ekf_params* models, int32_t n_models, const int32_t* model_of,
                                         int n_steps, int32_t* status) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(n >= 0 && n_steps >= 1, "n < 0 or n_steps < 1");
  CRB_REQUIRE(n_models >= 1, "n_models < 1");
  if (n == 0) return CRB_OK;
  CRB_REQUIRE(x && P && z && u, "NULL array");
  CRB_REQUIRE(models && model_of, "NULL model table or model_of");
  const int rc = crb_require_device(__func__);
  if (rc != CRB_OK) return rc;
  CRB_DEVICE_GUARD(ctx);   // ctx->device is current for this call, the caller's device is restored after it
  return ekf_many_launch(ctx, ctx->stream, n, n, x, P, z, u, n, n_steps, models, n_models, model_of, status);
}
