// crb_ekf_common.cuh — the EKF step's per-agent arithmetic and access helpers, shared by the single-model
// kernels (crb_ekf.cu) and the model-table kernels (crb_ekf_many.cu).  Both run this one ekf_step, which is what
// makes an agent of the model-table entry bitwise the single-model entry run with its model.
#pragma once
#include <stdint.h>

#include "crb_common.cuh"

// The constants of one step, in crb_ekf_params' layout (dt at 0, Q at 8, R at 72; 88 bytes).  The name is part of
// the single-model kernels' mangled names.
struct EkfArgs {
  double dt;
  float Q[16];
  float R[4];
};
static_assert(sizeof(EkfArgs) == sizeof(crb_ekf_params), "EkfArgs must have crb_ekf_params' layout");

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

// The model-table launch (crb_ekf_many.cu): agent i steps with models[model_of[i]].  Declared here because the
// resident track (crb_ekf.cu) runs it too.
int ekf_many_launch(crb_ctx* ctx, cudaStream_t st, int64_t count, int64_t ld, float* x, float* P, const float* z,
                    const float* u, int64_t ld_zu, int n_steps, const crb_ekf_params* models, int32_t n_models,
                    const int32_t* model_of, int32_t* status);
