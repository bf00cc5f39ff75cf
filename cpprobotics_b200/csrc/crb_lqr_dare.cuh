// crb_lqr_dare.cuh — the reference's fixed-point DARE iteration and LQR gain for one agent in registers, shared by
// crb_lqr_dlqr_kernel (crb_lqr.cu) and the path-tracking kernels (crb_lqr_track.cu).
//
// Replaces solve_DARE() + dlqr() of src/lqr_steer_control.cpp:75-96 (nx = 4, nu = 1, scalar R) and
// src/lqr_speed_steer_control.cpp:85-106 (nx = 5, nu = 2, 2x2 R).  Column-major matrices like Eigen: M(r,c) is
// element r + rows*c.  Pure FMA-pipe arithmetic, no transcendental: with -fmad=false and the reference's evaluation
// order (left to right, sequential-k sums, true division) the result is bit-identical to the CPU restatement,
// iteration counts included.
#pragma once
#include "crb_common.cuh"

template <int RA, int CA, int CB>
__device__ __forceinline__ void mm(const float (&A)[RA * CA], const float (&B)[CA * CB],
                                   float (&C)[RA * CB]) {
#pragma unroll
  for (int j = 0; j < CB; ++j)
#pragma unroll
    for (int i = 0; i < RA; ++i) {
      float s = A[i + RA * 0] * B[0 + CA * j];
#pragma unroll
      for (int k = 1; k < CA; ++k) s = s + A[i + RA * k] * B[k + CA * j];
      C[i + RA * j] = s;
    }
}

// solve_DARE then dlqr's gain.  X enters as anything and leaves as the returned X; K is nu x nx.  Returns the
// iterations executed; *converged says whether max|Xn - X| < eps ended them (the reference then returns Xn; after
// maxiter iterations without that it returns the last X, which is what X holds either way).
template <int NX, int NU>
__device__ __forceinline__ int crb_lqr_dlqr(const float (&A)[NX * NX], const float (&B)[NX * NU],
                                            const float (&Q)[NX * NX], const float (&R)[NU * NU], int maxiter,
                                            float eps, float (&K)[NX * NU], float (&X)[NX * NX], bool* converged) {
  constexpr int NN = NX * NX, NB = NX * NU;
  float At[NN], Bt[NB];
#pragma unroll
  for (int f = 0; f < NN; ++f) X[f] = Q[f];
#pragma unroll
  for (int r = 0; r < NX; ++r) {
#pragma unroll
    for (int c = 0; c < NX; ++c) At[c + NX * r] = A[r + NX * c];
#pragma unroll
    for (int c = 0; c < NU; ++c) Bt[c + NU * r] = B[r + NX * c];
  }
  bool conv = false;
  int it = 0;
  for (; it < maxiter; ++it) {  // solve_DARE :80-88 / :90-98
    float M1[NN], T1[NN], V1[NB], V2[NB], BtX[NB], S[NU * NU], M2[NN], M3[NN], T2[NN];
    mm<NX, NX, NX>(At, X, M1);
    mm<NX, NX, NX>(M1, A, T1);
    mm<NX, NX, NU>(M1, B, V1);
    mm<NU, NX, NX>(Bt, X, BtX);
    mm<NU, NX, NU>(BtX, B, S);
    if (NU == 1) {
      const float s = R[0] + S[0];
#pragma unroll
      for (int k = 0; k < NX; ++k) V2[k] = V1[k] / s;
    } else {
      float Sr[4], Sinv[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) Sr[k] = R[k % (NU * NU)] + S[k % (NU * NU)];
      const float det = Sr[0] * Sr[3] - Sr[1] * Sr[2];
      const float invdet = 1.0f / det;
      Sinv[0] = Sr[3] * invdet; Sinv[1] = -Sr[1] * invdet; Sinv[2] = -Sr[2] * invdet; Sinv[3] = Sr[0] * invdet;
      float V1b[NX * 2], V2b[NX * 2];
#pragma unroll
      for (int k = 0; k < NX * 2; ++k) V1b[k] = V1[k % NB];
      mm<NX, 2, 2>(V1b, Sinv, V2b);
#pragma unroll
      for (int k = 0; k < NB; ++k) V2[k] = V2b[k];
    }
    mm<NX, NU, NX>(V2, Bt, M2);
    mm<NX, NX, NX>(M2, X, M3);
    mm<NX, NX, NX>(M3, A, T2);
    float maxerr = 0.0f;
    float Xn[NN];
#pragma unroll
    for (int f = 0; f < NN; ++f) {
      Xn[f] = (T1[f] - T2[f]) + Q[f];
      const float e = fabsf(Xn[f] - X[f]);
      maxerr = (f == 0 || e > maxerr) ? e : maxerr;
    }
#pragma unroll
    for (int f = 0; f < NN; ++f) X[f] = Xn[f];
    if (maxerr < eps) { ++it; conv = true; break; }
  }
  // dlqr :92-96 / :102-106
  float BtX[NB], S[NU * NU], BtXA[NB];
  mm<NU, NX, NX>(Bt, X, BtX);
  mm<NU, NX, NU>(BtX, B, S);
  mm<NU, NX, NX>(BtX, A, BtXA);
  if (NU == 1) {
    const float s2 = S[0] + R[0];
    const float inv = (float)(1.0 / (double)s2);
#pragma unroll
    for (int j = 0; j < NX; ++j) K[j] = inv * BtXA[j];
  } else {
    float Sr[4], Sinv[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) Sr[k] = S[k % (NU * NU)] + R[k % (NU * NU)];
    const float det = Sr[0] * Sr[3] - Sr[1] * Sr[2];
    const float invdet = 1.0f / det;
    Sinv[0] = Sr[3] * invdet; Sinv[1] = -Sr[1] * invdet; Sinv[2] = -Sr[2] * invdet; Sinv[3] = Sr[0] * invdet;
    float Kb[2 * NX], Ab[2 * NX];
#pragma unroll
    for (int k = 0; k < 2 * NX; ++k) Ab[k] = BtXA[k % NB];
    mm<2, 2, NX>(Sinv, Ab, Kb);
#pragma unroll
    for (int k = 0; k < NB; ++k) K[k] = Kb[k];
  }
  *converged = conv;
  return it;
}
