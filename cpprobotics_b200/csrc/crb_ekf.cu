// crb_ekf.cu — batched EKF localisation step for sm_90a.
//
// Replaces ekf_estimation() of the reference, src/extended_kalman_filter.cpp:64-78, together with
// motion_model :22-36, jacobF :38-47, observation_model :50-55 and jacobH :57-62, for n independent
// agents per launch.
//
// Mapping: ONE THREAD PER AGENT.  The filter is a pure streaming op (176 algorithmic bytes and
// ~250 flops per update): the roofline is HBM, so what matters is that every warp-level access is
// one fully used 128-byte line.  All arrays are SoA field-major (field f of agent i at f*ld + i),
// so lane l of a warp reads consecutive floats of one field; the 24 loads of an agent are issued
// back to back (independent, ~96 B in flight per thread) and the 4x4 algebra lives in registers.
//
// Arithmetic: the kernel reproduces the dense Eigen evaluation of the reference entry for entry.
// jF is identity plus four entries and jH is a row selector; for finite operands, multiplying by an exact
// 0/1 and adding the resulting zero leaves a nonzero sum unchanged, so only the non-trivial terms are
// evaluated, in the same (sequential-k) order and with separate multiply and add (this TU is compiled with
// -fmad=false; the kernel is memory-bound, FMUL+FADD instead of FFMA costs nothing).  sin / cos carry the
// host libm's bits at every argument (crb_sincosf_libm), so every result is bit-identical to the CPU
// restatement on a host whose glibc runs its FMA build, with two exceptions the skipped terms cause: an
// exact zero may have the other sign (a dense sum adds +0 terms, turning -0 into +0), and in an agent with
// an infinite input the dense 0 * inf makes NaN of every entry, also of those this kernel computes without
// that input (tests/test_ekf_edges.py).
#include <stdint.h>

#include "crb_ekf_common.cuh"

// count agents, leading dimension ld (>= count) for x/P, ld_zu for z/u (they may live in a staging
// buffer with a different pitch).  Each thread filters V consecutive agents; V = 2 needs count, ld and ld_zu
// even and 8-byte aligned arrays (ekf_launch checks), and then a warp access is 256 contiguous bytes of one
// field: half the memory instructions per byte, and the two agents' algebra is independent work for the
// scheduler while their loads are in flight.
template <int BLOCK, int MINB, int V>
__global__ void __launch_bounds__(BLOCK, MINB)
crb_ekf_step_kernel(int64_t count, int64_t ld, float* __restrict__ x, float* __restrict__ P,
                    const float* __restrict__ z, const float* __restrict__ u, int64_t ld_zu,
                    int n_steps, EkfArgs a) {
  const int64_t i = V * ((int64_t)blockIdx.x * blockDim.x + threadIdx.x);
  if (i >= count) return;
  crb_pdl_launch_dependents();   // the next launch may start scheduling its CTAs behind ours
  crb_pdl_wait();   // the previous launch on this stream (e.g. the preceding filter step) is complete
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
      ekf_step(xk, Pk, z0[k], z1[k], u0[k], u1[k], a);
#pragma unroll
      for (int f = 0; f < 4; ++f) xs[f][k] = xk[f];
#pragma unroll
      for (int f = 0; f < 16; ++f) Ps[f][k] = Pk[f];
      z0[k] = nz0[k]; z1[k] = nz1[k]; u0[k] = nu0[k]; u1[k] = nu1[k];
    }
  }
  // The store addresses are recomputed after the math instead of reusing the load addresses: keeping ~20
  // 64-bit field addresses live across ekf_step costs 80 registers and a 24-byte spill on the hot path.  The
  // empty asm hides that ld and i are the values the loads used.  Offsets stay 64-bit: 19 * ld + i passes 2^31
  // at about 1.1e8 agents.
  int64_t lds = ld, is = i;
  asm volatile("" : "+l"(lds), "+l"(is));
#pragma unroll
  for (int f = 0; f < 4; ++f) st_agents<V>(x + f * lds + is, xs[f]);
#pragma unroll
  for (int f = 0; f < 16; ++f) st_agents<V>(P + f * lds + is, Ps[f]);
}

static int ekf_launch(crb_ctx* ctx, cudaStream_t st, int64_t count, int64_t ld, float* x, float* P,
                      const float* z, const float* u, int64_t ld_zu, int n_steps,
                      const crb_ekf_params* prm) {
  EkfArgs a;
  a.dt = prm->dt;
  memcpy(a.Q, prm->Q, sizeof(a.Q));
  memcpy(a.R, prm->R, sizeof(a.R));
  // Launch shape: two agents per thread in 128-thread CTAs, 4 resident per SM, whenever the arrays allow 8-byte
  // accesses; otherwise one agent per thread in 256-thread CTAs, 3 per SM.  Either way every SM has ~24 KB of
  // independent reads in flight per 256 agents, which covers H100's HBM latency.  Measured at 2^20 agents, 30
  // graph-captured launches over 3 buffer sets, on two H100 80GB HBM3 boxes (700 W limit): the two-agent form runs
  // 4.6 % and 6.4 % faster than the one-agent form, and 4, 2 or 6 CTAs per SM make no difference (DESIGN.md 3).
  // two agents per thread: every row segment a thread touches is 8-byte aligned
  const bool pair_ok = (count % 2) == 0 && (ld % 2) == 0 && (ld_zu % 2) == 0 &&
                       (((uintptr_t)x | (uintptr_t)P | (uintptr_t)z | (uintptr_t)u) & 7) == 0;
  if (pair_ok)
    CRB_CUDA(crb_launch_pdl(crb_ekf_step_kernel<128, 4, 2>, (unsigned)crb_grid_for(count / 2, 128), 128u, st,
                            count, ld, x, P, z, u, ld_zu, n_steps, a));
  else
    CRB_CUDA(crb_launch_pdl(crb_ekf_step_kernel<256, 3, 1>, (unsigned)crb_grid_for(count, 256), 256u, st,
                            count, ld, x, P, z, u, ld_zu, n_steps, a));
  ctx->launches++;
  return CRB_OK;
}

extern "C" int crb_ekf_step_batched(crb_ctx* ctx, int64_t n, float* x, float* P, const float* z,
                                    const float* u, const crb_ekf_params* prm, int n_steps) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_DEVICE_GUARD(ctx);   // ctx->device is current for this call, the caller's device is restored after it
  CRB_REQUIRE(n >= 0 && n_steps >= 1, "n < 0 or n_steps < 1");
  CRB_REQUIRE(prm != nullptr, "prm is NULL");
  if (n == 0) return CRB_OK;
  CRB_REQUIRE(x && P && z && u, "NULL array");
  return ekf_launch(ctx, ctx->stream, n, n, x, P, z, u, n, n_steps, prm);
}

// Host-pointer variant: chunks of agents stream through CRB_N_PIPE staging arenas, each on its own
// stream (H2D chunk k+1 and D2H chunk k-1 overlap the kernel of chunk k: both copy engines busy).
constexpr int64_t EKF_HOST_CHUNK = 131072;  // agents per chunk
extern "C" int crb_ekf_step_batched_host(crb_ctx* ctx, int64_t n, float* x, float* P,
                                         const float* z, const float* u,
                                         const crb_ekf_params* prm, int n_steps) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(n >= 0 && n_steps >= 1, "n < 0 or n_steps < 1");
  CRB_REQUIRE(prm != nullptr, "prm is NULL");
  if (n == 0) return CRB_OK;
  CRB_REQUIRE(x && P && z && u, "NULL array");
  CRB_CUDA(cudaSetDevice(ctx->device));
  // Pinned + mapped buffers: run the resident kernel on them directly (see crb_host_mapped).
  if (crb_zero_copy_enabled()) {
    float *mx, *mP;
    const float *mz, *mu;
    if (crb_host_mapped(x, &mx) && crb_host_mapped(P, &mP) && crb_host_mapped(z, &mz) &&
        crb_host_mapped(u, &mu)) {
      cudaStream_t st = ctx->pipe_stream[0];
      int rc = ekf_launch(ctx, st, n, n, mx, mP, mz, mu, n, n_steps, prm);
      if (rc) return rc;
      CRB_CUDA(cudaStreamSynchronize(st));
      return CRB_OK;
    }
  }
  const int64_t chunk_cap = n < EKF_HOST_CHUNK ? n : EKF_HOST_CHUNK;
  const size_t nf = 20 + (size_t)4 * n_steps;  // x4 P16 z2s u2s
  const size_t pitch = (size_t)chunk_cap * sizeof(float);
  for (int s = 0; s < CRB_N_PIPE; ++s) {
    int rc = crb_ctx_pipe_reserve(ctx, s, nf * pitch);
    if (rc) return rc;
  }
  const size_t hp = (size_t)n * sizeof(float);
  int slot = 0;
  for (int64_t i0 = 0; i0 < n; i0 += chunk_cap, slot = (slot + 1) % CRB_N_PIPE) {
    const int64_t cnt = (n - i0) < chunk_cap ? (n - i0) : chunk_cap;
    cudaStream_t st = ctx->pipe_stream[slot];
    float* dx = (float*)ctx->pipe_buf[slot];
    float* dP = dx + 4 * chunk_cap;
    float* dz = dP + 16 * chunk_cap;
    float* du = dz + (size_t)2 * n_steps * chunk_cap;
    const size_t w = (size_t)cnt * sizeof(float);
    CRB_CUDA(crb_copy_rows(dx, pitch, x + i0, hp, w, 4, cudaMemcpyHostToDevice, st));
    CRB_CUDA(crb_copy_rows(dP, pitch, P + i0, hp, w, 16, cudaMemcpyHostToDevice, st));
    CRB_CUDA(crb_copy_rows(dz, pitch, z + i0, hp, w, (size_t)2 * n_steps,
                               cudaMemcpyHostToDevice, st));
    CRB_CUDA(crb_copy_rows(du, pitch, u + i0, hp, w, (size_t)2 * n_steps,
                               cudaMemcpyHostToDevice, st));
    int rc = ekf_launch(ctx, st, cnt, chunk_cap, dx, dP, dz, du, chunk_cap, n_steps, prm);
    if (rc) return rc;
    CRB_CUDA(crb_copy_rows(x + i0, hp, dx, pitch, w, 4, cudaMemcpyDeviceToHost, st));
    CRB_CUDA(crb_copy_rows(P + i0, hp, dP, pitch, w, 16, cudaMemcpyDeviceToHost, st));
  }
  for (int s = 0; s < CRB_N_PIPE; ++s) CRB_CUDA(cudaStreamSynchronize(ctx->pipe_stream[s]));
  return CRB_OK;
}


// ---- resident-state tracking: the reference's own time loop ----------------------------------------------
// src/extended_kalman_filter.cpp:171-183 keeps xEst, PEst across iterations and receives only (z, u) per step.
// crb_ekf_step_batched_host ships all 176 bytes per update every call, which pins the end-to-end rate to the
// PCIe link (96 B in + 80 B out).  A track keeps x and P in HBM; a step ships 16 B in (z, u) and, if asked,
// 16 B out (x).  Pinned + mapped z / u are read by the kernel straight over PCIe; x goes back through a
// device-side snapshot on a second stream, so the D2H copy of step k overlaps the kernel of step k+1 (the two
// directions of the link at once).
struct crb_ekf_track {
  int64_t n;
  float* x;        // [4][n]
  float* P;        // [16][n]
  float* snap[2];  // [4][n] each: x of the last two steps on their way to the host
  float* stage;    // [4][n]: z, u staging for pageable callers (allocated on first use)
  cudaEvent_t ev_kernel[2], ev_copy[2];
  int parity;
  int64_t steps;
};

extern "C" int crb_ekf_track_open(crb_ctx* ctx, int64_t n, const float* x0_host, const float* P0_host,
                                  crb_ekf_track** out) {
  CRB_REQUIRE(ctx != nullptr && out != nullptr, "ctx / out is NULL");
  CRB_REQUIRE(n > 0 && x0_host && P0_host, "n <= 0 or NULL initial state");
  CRB_DEVICE_GUARD(ctx);
  *out = nullptr;
  crb_ekf_track* t = new crb_ekf_track();
  memset(t, 0, sizeof(*t));
  t->n = n;
  const size_t row = (size_t)n * sizeof(float);
  cudaError_t e = cudaMalloc(&t->x, 4 * row);
  if (e == cudaSuccess) e = cudaMalloc(&t->P, 16 * row);
  for (int k = 0; k < 2 && e == cudaSuccess; ++k) e = cudaMalloc(&t->snap[k], 4 * row);
  for (int k = 0; k < 2 && e == cudaSuccess; ++k) e = cudaEventCreateWithFlags(&t->ev_kernel[k], cudaEventDisableTiming);
  for (int k = 0; k < 2 && e == cudaSuccess; ++k) e = cudaEventCreateWithFlags(&t->ev_copy[k], cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaMemcpy(t->x, x0_host, 4 * row, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(t->P, P0_host, 16 * row, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    crb_set_error("crb_ekf_track_open: %s", cudaGetErrorString(e));
    crb_ekf_track_close(ctx, t);
    return e == cudaErrorMemoryAllocation ? CRB_ERR_ALLOC : CRB_ERR_CUDA;
  }
  *out = t;
  return CRB_OK;
}

extern "C" int crb_ekf_track_close(crb_ctx* ctx, crb_ekf_track* t) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  if (!t) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  cudaStreamSynchronize(ctx->pipe_stream[0]);
  cudaStreamSynchronize(ctx->pipe_stream[1]);
  if (t->x) cudaFree(t->x);
  if (t->P) cudaFree(t->P);
  for (int k = 0; k < 2; ++k) {
    if (t->snap[k]) cudaFree(t->snap[k]);
    if (t->ev_kernel[k]) cudaEventDestroy(t->ev_kernel[k]);
    if (t->ev_copy[k]) cudaEventDestroy(t->ev_copy[k]);
  }
  if (t->stage) cudaFree(t->stage);
  delete t;
  return CRB_OK;
}

extern "C" int crb_ekf_track_sync(crb_ctx* ctx, crb_ekf_track* t) {
  CRB_REQUIRE(ctx != nullptr && t != nullptr, "ctx / track is NULL");
  CRB_DEVICE_GUARD(ctx);
  CRB_CUDA(cudaStreamSynchronize(ctx->pipe_stream[0]));
  CRB_CUDA(cudaStreamSynchronize(ctx->pipe_stream[1]));
  return CRB_OK;
}

// One step of a track: z, u reach the device (in place when pinned and mapped, else through t->stage), launch(sk, mz,
// mu) enqueues the step on the track's kernel stream, and x goes out through the snapshot rotation.  The entry points
// below differ only in that launch.
template <class Launch>
static int ekf_track_step_body(crb_ctx* ctx, crb_ekf_track* t, const float* z_host, const float* u_host,
                               float* x_out_host, int async, Launch&& launch) {
  const int64_t n = t->n;
  const size_t row = (size_t)n * sizeof(float);
  cudaStream_t sk = ctx->pipe_stream[0], sc = ctx->pipe_stream[1];
  const int p = t->parity;
  const float *mz = nullptr, *mu = nullptr;
  const bool direct = crb_zero_copy_enabled() && crb_host_mapped(z_host, &mz) && crb_host_mapped(u_host, &mu);
  if (!direct) {  // pageable (or zero-copy disabled): stage z, u through the device
    if (!t->stage) CRB_CUDA(cudaMalloc(&t->stage, 4 * row));
    CRB_CUDA(cudaMemcpyAsync(t->stage, z_host, 2 * row, cudaMemcpyHostToDevice, sk));
    CRB_CUDA(cudaMemcpyAsync(t->stage + 2 * n, u_host, 2 * row, cudaMemcpyHostToDevice, sk));
    mz = t->stage;
    mu = t->stage + 2 * n;
  }
  int rc = launch(sk, mz, mu);
  if (rc) return rc;
  if (x_out_host) {
    // snapshot p was last used two steps ago: its copy must have left before it is overwritten
    if (t->steps >= 2) CRB_CUDA(cudaStreamWaitEvent(sk, t->ev_copy[p], 0));
    CRB_CUDA(cudaMemcpyAsync(t->snap[p], t->x, 4 * row, cudaMemcpyDeviceToDevice, sk));
    CRB_CUDA(cudaEventRecord(t->ev_kernel[p], sk));
    CRB_CUDA(cudaStreamWaitEvent(sc, t->ev_kernel[p], 0));
    CRB_CUDA(cudaMemcpyAsync(x_out_host, t->snap[p], 4 * row, cudaMemcpyDeviceToHost, sc));
    CRB_CUDA(cudaEventRecord(t->ev_copy[p], sc));
    t->parity ^= 1;
    t->steps++;
  }
  if (!async) {
    CRB_CUDA(cudaStreamSynchronize(sk));
    CRB_CUDA(cudaStreamSynchronize(sc));
  }
  return CRB_OK;
}

extern "C" int crb_ekf_track_step(crb_ctx* ctx, crb_ekf_track* t, const float* z_host, const float* u_host,
                                  const crb_ekf_params* prm, float* x_out_host, int async) {
  CRB_REQUIRE(ctx != nullptr && t != nullptr && prm != nullptr, "ctx / track / prm is NULL");
  CRB_REQUIRE(z_host && u_host, "NULL observation / control array");
  CRB_DEVICE_GUARD(ctx);
  return ekf_track_step_body(ctx, t, z_host, u_host, x_out_host, async,
                             [&](cudaStream_t sk, const float* mz, const float* mu) {
                               return ekf_launch(ctx, sk, t->n, t->n, t->x, t->P, mz, mu, t->n, 1, prm);
                             });
}

extern "C" int crb_ekf_track_step_many(crb_ctx* ctx, crb_ekf_track* t, const float* z_host, const float* u_host,
                                       const crb_ekf_params* models, int32_t n_models, const int32_t* model_of,
                                       int32_t* status, float* x_out_host, int async) {
  CRB_REQUIRE(ctx != nullptr && t != nullptr, "ctx / track is NULL");
  CRB_REQUIRE(z_host && u_host, "NULL observation / control array");
  CRB_REQUIRE(models && model_of && n_models >= 1, "NULL model table / model_of, or n_models < 1");
  CRB_DEVICE_GUARD(ctx);
  return ekf_track_step_body(ctx, t, z_host, u_host, x_out_host, async,
                             [&](cudaStream_t sk, const float* mz, const float* mu) {
                               return ekf_many_launch(ctx, sk, t->n, t->n, t->x, t->P, mz, mu, t->n, 1, models,
                                                      n_models, model_of, status);
                             });
}

extern "C" int crb_ekf_track_read(crb_ctx* ctx, crb_ekf_track* t, float* x_host, float* P_host) {
  CRB_REQUIRE(ctx != nullptr && t != nullptr, "ctx / track is NULL");
  CRB_DEVICE_GUARD(ctx);
  const size_t row = (size_t)t->n * sizeof(float);
  CRB_CUDA(cudaStreamSynchronize(ctx->pipe_stream[0]));
  CRB_CUDA(cudaStreamSynchronize(ctx->pipe_stream[1]));
  if (x_host) CRB_CUDA(cudaMemcpy(x_host, t->x, 4 * row, cudaMemcpyDeviceToHost));
  if (P_host) CRB_CUDA(cudaMemcpy(P_host, t->P, 16 * row, cudaMemcpyDeviceToHost));
  return CRB_OK;
}
