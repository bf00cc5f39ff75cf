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
#include <stdlib.h>

#include "crb_common.cuh"

struct EkfArgs {
  double dt;
  float Q[16];
  float R[4];
};

// One filter step on register state.  P is column-major: P[r + 4*c].
__device__ __forceinline__ void ekf_step(float (&x)[4], float (&P)[16], float z0, float z1,
                                         float u0, float u1, const EkfArgs& a) {
  // ---- motion_model(xEst, u) :22-36.  B_(0,0) = DT*cos(yaw) is a double product narrowed to float.
  float s, c;
  crb_sincosf_libm(x[2], s, c);   // the host libm's bits (crb_common.cuh)
  const float b00 = (float)(a.dt * (double)c);
  const float b10 = (float)(a.dt * (double)s);
  const float b21 = (float)a.dt;
  float xp[4];
  xp[0] = x[0] + b00 * u0;
  xp[1] = x[1] + b10 * u0;
  xp[2] = x[2] + b21 * u1;
  xp[3] = x[3] + u0;  // F_(3,3) = 1 and B_(3,0) = 1: v accumulates (reference quirk)

  // ---- jacobF(xPred, u) :38-47: evaluated at the PREDICTED yaw with v = u(0).
  float s2, c2;
  crb_sincosf_libm(xp[2], s2, c2);
  const float j02 = (float)((-a.dt * (double)u0) * (double)s2);
  const float j03 = (float)(a.dt * (double)c2);
  const float j12 = (float)((a.dt * (double)u0) * (double)c2);
  const float j13 = (float)(a.dt * (double)s2);

  // ---- PPred = (jF*P)*jF^T + Q :69.
  // T = jF*P: rows 2,3 are rows of P; row 0 = (P0j + j02*P2j) + j03*P3j; row 1 likewise.
  float T[16];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    T[0 + 4 * j] = (P[0 + 4 * j] + j02 * P[2 + 4 * j]) + j03 * P[3 + 4 * j];
    T[1 + 4 * j] = (P[1 + 4 * j] + j12 * P[2 + 4 * j]) + j13 * P[3 + 4 * j];
    T[2 + 4 * j] = P[2 + 4 * j];
    T[3 + 4 * j] = P[3 + 4 * j];
  }
  // PP = T*jF^T + Q: columns 2,3 are columns of T; column 0 = (Ti0 + Ti2*j02) + Ti3*j03.
  float PP[16];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    PP[i + 4 * 0] = ((T[i + 4 * 0] + T[i + 4 * 2] * j02) + T[i + 4 * 3] * j03) + a.Q[i + 4 * 0];
    PP[i + 4 * 1] = ((T[i + 4 * 1] + T[i + 4 * 2] * j12) + T[i + 4 * 3] * j13) + a.Q[i + 4 * 1];
    PP[i + 4 * 2] = T[i + 4 * 2] + a.Q[i + 4 * 2];
    PP[i + 4 * 3] = T[i + 4 * 3] + a.Q[i + 4 * 3];
  }

  // ---- update :71-77.  zPred = xPred.xy; S = PPred[0:2,0:2] + R; closed-form 2x2 inverse.
  const float y0 = z0 - xp[0];
  const float y1 = z1 - xp[1];
  const float S00 = PP[0] + a.R[0], S10 = PP[1] + a.R[1];
  const float S01 = PP[4] + a.R[2], S11 = PP[5] + a.R[3];
  const float det = S00 * S11 - S10 * S01;
  const float invdet = 1.0f / det;
  const float i00 = S11 * invdet, i10 = -S10 * invdet;
  const float i01 = -S01 * invdet, i11 = S00 * invdet;
  float K0[4], K1[4];  // K = (PPred*jH^T) * S^-1, columns 0 and 1
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    K0[i] = PP[i] * i00 + PP[i + 4] * i10;
    K1[i] = PP[i] * i01 + PP[i + 4] * i11;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) x[i] = xp[i] + (K0[i] * y0 + K1[i] * y1);
  // PEst = (I - K*jH)*PPred: M = I - K*jH has columns (e0-K0, e1-K1, e2, e3).
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float p0 = PP[0 + 4 * j], p1 = PP[1 + 4 * j];
    P[0 + 4 * j] = (1.0f - K0[0]) * p0 + (0.0f - K1[0]) * p1;
    P[1 + 4 * j] = (0.0f - K0[1]) * p0 + (1.0f - K1[1]) * p1;
    P[2 + 4 * j] = ((0.0f - K0[2]) * p0 + (0.0f - K1[2]) * p1) + PP[2 + 4 * j];
    P[3 + 4 * j] = ((0.0f - K0[3]) * p0 + (0.0f - K1[3]) * p1) + PP[3 + 4 * j];
  }
}

// V consecutive floats of one field: one 4-byte (V = 1) or 8-byte (V = 2) streaming access.
template <int V>
__device__ __forceinline__ void ld_agents(const float* p, float (&v)[V]) {
  if constexpr (V == 1) {
    v[0] = ld_stream(p);
  } else {
    const float2 t = __ldcs(reinterpret_cast<const float2*>(p));
    v[0] = t.x;
    v[1] = t.y;
  }
}
template <int V>
__device__ __forceinline__ void st_agents(float* p, const float (&v)[V]) {
  if constexpr (V == 1) st_stream(p, v[0]);
  else __stcs(reinterpret_cast<float2*>(p), make_float2(v[0], v[1]));
}

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

// ---------------------------------------------------------------------------------------------------
// TMA-staged variant (CRB_EKF_VARIANT=4): persistent CTAs, each tile of EKF_TILE agents is brought into
// shared memory by 24 bulk async copies (cp.async.bulk, one 512-byte row segment per field; SASS: UBLKCP)
// that complete on an mbarrier, EKF_STAGES tiles deep, and leaves through 20 bulk stores.  Loads of
// tile k+S are in flight while tile k is computed without holding registers.  A/B against the
// direct-load kernel in DESIGN.md 3.
// ---------------------------------------------------------------------------------------------------
#define EKF_NIN 24
#define EKF_NOUT 20

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  }
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst_smem)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* dst, const void* src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst),
               "r"(smem_u32(src_smem)), "r"(bytes)
               : "memory");
}

template <int EKF_TILE, int EKF_STAGES>
__global__ void __launch_bounds__(EKF_TILE)
crb_ekf_step_tma_kernel(int64_t count, int64_t ld, float* __restrict__ x, float* __restrict__ P,
                        const float* __restrict__ z, const float* __restrict__ u, int64_t ld_zu,
                        EkfArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* sin_ = (float*)smem_raw;                                        // [STAGES][NIN][TILE]
  float* sout = sin_ + EKF_STAGES * EKF_NIN * EKF_TILE;                  // [2][NOUT][TILE]
  uint64_t* full = (uint64_t*)(sout + 2 * EKF_NOUT * EKF_TILE);          // [STAGES]
  const int tid = threadIdx.x;
  const int64_t ntiles = (count + EKF_TILE - 1) / EKF_TILE;
  if (tid == 0) {
    for (int s = 0; s < EKF_STAGES; ++s) mbar_init(&full[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  auto issue_loads = [&](int64_t tile, int stage) {  // thread 0 only
    const int64_t i0 = tile * EKF_TILE;
    const uint32_t cnt = (uint32_t)((count - i0) < EKF_TILE ? (count - i0) : EKF_TILE);
    const uint32_t bytes = cnt * 4u;
    float* dst = sin_ + (size_t)stage * EKF_NIN * EKF_TILE;
    mbar_expect_tx(&full[stage], bytes * EKF_NIN);
#pragma unroll
    for (int f = 0; f < 4; ++f) bulk_g2s(dst + f * EKF_TILE, x + f * ld + i0, bytes, &full[stage]);
#pragma unroll
    for (int f = 0; f < 16; ++f)
      bulk_g2s(dst + (4 + f) * EKF_TILE, P + f * ld + i0, bytes, &full[stage]);
#pragma unroll
    for (int f = 0; f < 2; ++f) {
      bulk_g2s(dst + (20 + f) * EKF_TILE, z + f * ld_zu + i0, bytes, &full[stage]);
      bulk_g2s(dst + (22 + f) * EKF_TILE, u + f * ld_zu + i0, bytes, &full[stage]);
    }
  };

  // prologue: fill the pipeline
  if (tid == 0) {
    for (int s = 0; s < EKF_STAGES; ++s) {
      const int64_t t = (int64_t)blockIdx.x + (int64_t)s * gridDim.x;
      if (t < ntiles) issue_loads(t, s);
    }
  }
  int k = 0;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++k) {
    const int stage = k % EKF_STAGES;
    const uint32_t parity = (uint32_t)((k / EKF_STAGES) & 1);
    const int ob = k & 1;
    const int64_t i0 = tile * EKF_TILE;
    const bool active = i0 + tid < count;
    mbar_wait(&full[stage], parity);
    const float* si = sin_ + (size_t)stage * EKF_NIN * EKF_TILE + tid;
    float xs[4], Ps[16];
#pragma unroll
    for (int f = 0; f < 4; ++f) xs[f] = si[f * EKF_TILE];
#pragma unroll
    for (int f = 0; f < 16; ++f) Ps[f] = si[(4 + f) * EKF_TILE];
    const float z0 = si[20 * EKF_TILE], z1 = si[21 * EKF_TILE];
    const float u0 = si[22 * EKF_TILE], u1 = si[23 * EKF_TILE];
    // the bulk store issued two tiles ago must have finished READING sout[ob] before it is rewritten
    if (tid == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
    __syncthreads();  // every thread has its inputs in registers: the stage can be refilled
    if (tid == 0) {
      const int64_t nt = tile + (int64_t)EKF_STAGES * gridDim.x;
      if (nt < ntiles) issue_loads(nt, stage);
    }
    if (active) ekf_step(xs, Ps, z0, z1, u0, u1, a);
    float* so = sout + (size_t)ob * EKF_NOUT * EKF_TILE + tid;
#pragma unroll
    for (int f = 0; f < 4; ++f) so[f * EKF_TILE] = xs[f];
#pragma unroll
    for (int f = 0; f < 16; ++f) so[(4 + f) * EKF_TILE] = Ps[f];
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic writes -> async proxy
    __syncthreads();
    if (tid == 0) {
      const uint32_t cnt = (uint32_t)((count - i0) < EKF_TILE ? (count - i0) : EKF_TILE);
      const uint32_t bytes = cnt * 4u;
      const float* src = sout + (size_t)ob * EKF_NOUT * EKF_TILE;
#pragma unroll
      for (int f = 0; f < 4; ++f) bulk_s2g(x + f * ld + i0, src + f * EKF_TILE, bytes);
#pragma unroll
      for (int f = 0; f < 16; ++f) bulk_s2g(P + f * ld + i0, src + (4 + f) * EKF_TILE, bytes);
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
  }
  if (tid == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

static size_t ekf_tma_smem_bytes(int tile, int stages) {
  return (size_t)(stages * EKF_NIN + 2 * EKF_NOUT) * tile * sizeof(float) + stages * sizeof(uint64_t);
}

template <int TILE, int STAGES>
static int ekf_tma_launch(crb_ctx* ctx, cudaStream_t st, int64_t count, int64_t ld, float* x,
                          float* P, const float* z, const float* u, int64_t ld_zu,
                          const EkfArgs& a) {
  // per-context latch (bit per instantiation): the attribute is per device, and a process may hold contexts
  // on several devices
  const size_t smem = ekf_tma_smem_bytes(TILE, STAGES);
  const int bit = 1 << ((TILE == 256 ? 2 : 0) + (STAGES == 3 ? 1 : 0));
  if (!(ctx->ekf_tma_attr_set & bit)) {
    CRB_CUDA(cudaFuncSetAttribute(crb_ekf_step_tma_kernel<TILE, STAGES>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ctx->ekf_tma_attr_set |= bit;
  }
  const int64_t ntiles = (count + TILE - 1) / TILE;
  int per_sm = (int)((size_t)227 * 1024 / (smem + 1024));
  if (per_sm * TILE > 2048) per_sm = 2048 / TILE;
  int grid = ctx->sm_count * (per_sm > 0 ? per_sm : 1);
  if ((int64_t)grid > ntiles) grid = (int)ntiles;
  crb_ekf_step_tma_kernel<TILE, STAGES><<<grid, TILE, smem, st>>>(count, ld, x, P, z, u, ld_zu, a);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
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
  // CRB_EKF_VARIANT selects alternatives for A/B measurements.
  static int variant = -1;
  if (variant < 0) {
    const char* e = getenv("CRB_EKF_VARIANT");
    variant = e ? atoi(e) : 0;
  }
  // bulk copies need 16-byte aligned, 16-byte multiple row segments
  const bool tma_ok = n_steps == 1 && (ld % 4) == 0 && (ld_zu % 4) == 0 && (count % 4) == 0 &&
                      (((uintptr_t)x | (uintptr_t)P | (uintptr_t)z | (uintptr_t)u) & 15) == 0;
  // two agents per thread: every row segment a thread touches is 8-byte aligned
  const bool pair_ok = (count % 2) == 0 && (ld % 2) == 0 && (ld_zu % 2) == 0 &&
                       (((uintptr_t)x | (uintptr_t)P | (uintptr_t)z | (uintptr_t)u) & 7) == 0;
  if (tma_ok && variant == 4) return ekf_tma_launch<128, 3>(ctx, st, count, ld, x, P, z, u, ld_zu, a);
  if (tma_ok && variant == 5) return ekf_tma_launch<128, 2>(ctx, st, count, ld, x, P, z, u, ld_zu, a);
  if (tma_ok && variant == 6) return ekf_tma_launch<256, 2>(ctx, st, count, ld, x, P, z, u, ld_zu, a);
  if (tma_ok && variant == 7) return ekf_tma_launch<256, 3>(ctx, st, count, ld, x, P, z, u, ld_zu, a);
  switch (variant) {
    case 1:
      crb_ekf_step_kernel<256, 4, 1><<<crb_grid_for(count, 256), 256, 0, st>>>(count, ld, x, P, z, u,
                                                                            ld_zu, n_steps, a);
      break;
    case 2:
      crb_ekf_step_kernel<128, 8, 1><<<crb_grid_for(count, 128), 128, 0, st>>>(count, ld, x, P, z, u,
                                                                            ld_zu, n_steps, a);
      break;
    case 3:
      crb_ekf_step_kernel<512, 2, 1><<<crb_grid_for(count, 512), 512, 0, st>>>(count, ld, x, P, z, u,
                                                                            ld_zu, n_steps, a);
      break;
    default:
      if (pair_ok)
        CRB_CUDA(crb_launch_pdl(crb_ekf_step_kernel<128, 4, 2>, (unsigned)crb_grid_for(count / 2, 128), 128u, st,
                                count, ld, x, P, z, u, ld_zu, n_steps, a));
      else
        CRB_CUDA(crb_launch_pdl(crb_ekf_step_kernel<256, 3, 1>, (unsigned)crb_grid_for(count, 256), 256u, st,
                                count, ld, x, P, z, u, ld_zu, n_steps, a));
  }
  CRB_CUDA(cudaGetLastError());
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
  static int64_t chunk_pref = 0;  // CRB_EKF_CHUNK overrides the staging chunk (agents) for A/B
  if (chunk_pref == 0) {
    const char* e = getenv("CRB_EKF_CHUNK");
    chunk_pref = e ? atoll(e) : 131072;
    if (chunk_pref < 1024) chunk_pref = 131072;
  }
  const int64_t chunk_cap = n < chunk_pref ? n : chunk_pref;
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

extern "C" int crb_ekf_track_step(crb_ctx* ctx, crb_ekf_track* t, const float* z_host, const float* u_host,
                                  const crb_ekf_params* prm, float* x_out_host, int async) {
  CRB_REQUIRE(ctx != nullptr && t != nullptr && prm != nullptr, "ctx / track / prm is NULL");
  CRB_REQUIRE(z_host && u_host, "NULL observation / control array");
  CRB_DEVICE_GUARD(ctx);
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
  int rc = ekf_launch(ctx, sk, n, n, t->x, t->P, mz, mu, n, 1, prm);
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
