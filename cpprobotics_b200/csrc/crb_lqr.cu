// crb_lqr.cu — batched discrete LQR gain by the reference's fixed-point DARE iteration, for sm_90a.
//
// Replaces solve_DARE() + dlqr() of src/lqr_steer_control.cpp:75-96 (nx = 4, nu = 1, scalar R) and
// src/lqr_speed_steer_control.cpp:85-106 (nx = 5, nu = 2, 2x2 R) for n independent agents per launch
// (SURVEY.md §8 row f-4: the same small-matrix engine, time-invariant A, B).
//
// Mapping: one thread per agent, A / B / X and the temporaries in registers, SoA field-major arrays
// (column-major matrices like Eigen: M(r,c) is field r + nx*c).  Pure FMA-pipe arithmetic, no
// transcendental: with -fmad=false and the reference's evaluation order (left to right, sequential-k
// sums, true division) the result is bit-identical to the CPU restatement, iteration counts included.
#include "crb_lqr_dare.cuh"

template <int NX, int NU>
__global__ void __launch_bounds__(128)
crb_lqr_dlqr_kernel(int64_t n, const float* __restrict__ Ag, const float* __restrict__ Bg,
                    const float* __restrict__ Qg, const float* __restrict__ Rg, int maxiter,
                    float eps, float* __restrict__ Kg, float* __restrict__ Xg,
                    int32_t* __restrict__ itg) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  constexpr int NN = NX * NX, NB = NX * NU;
  float A[NN], B[NB], Q[NN], R[NU * NU], X[NN], K[NB];
#pragma unroll
  for (int f = 0; f < NN; ++f) { A[f] = Ag[(int64_t)f * n + i]; Q[f] = Qg[f]; }
#pragma unroll
  for (int f = 0; f < NB; ++f) B[f] = Bg[(int64_t)f * n + i];
#pragma unroll
  for (int f = 0; f < NU * NU; ++f) R[f] = Rg[f];
  bool converged;
  const int it = crb_lqr_dlqr<NX, NU>(A, B, Q, R, maxiter, eps, K, X, &converged);
#pragma unroll
  for (int f = 0; f < NB; ++f) Kg[(int64_t)f * n + i] = K[f];
  if (Xg) {
#pragma unroll
    for (int f = 0; f < NN; ++f) Xg[(int64_t)f * n + i] = X[f];
  }
  if (itg) itg[i] = it;
}

extern "C" int crb_lqr_dlqr_batched(crb_ctx* ctx, int64_t n, int nx, int nu, const float* A,
                                    const float* B, const float* Q, const float* R, int maxiter,
                                    float eps, float* K, float* X, int32_t* iters) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_DEVICE_GUARD(ctx);   // ctx->device is current for this call, the caller's device is restored after it
  CRB_REQUIRE(n >= 0 && maxiter >= 0, "n < 0 or maxiter < 0");
  CRB_REQUIRE((nx == 4 && nu == 1) || (nx == 5 && nu == 2),
              "supported shapes: (nx, nu) = (4, 1) [lqr_steer_control] or (5, 2) [lqr_speed_steer_control]");
  if (n == 0) return CRB_OK;
  CRB_REQUIRE(A && B && Q && R && K, "NULL array");
  const int block = 128;
  if (nx == 4)
    crb_lqr_dlqr_kernel<4, 1><<<crb_grid_for(n, block), block, 0, ctx->stream>>>(n, A, B, Q, R, maxiter,
                                                                                 eps, K, X, iters);
  else
    crb_lqr_dlqr_kernel<5, 2><<<crb_grid_for(n, block), block, 0, ctx->stream>>>(n, A, B, Q, R, maxiter,
                                                                                 eps, K, X, iters);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}
