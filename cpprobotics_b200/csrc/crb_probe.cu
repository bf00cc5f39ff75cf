// crb_probe.cu — measurement aids: the roofline denominators that MEASURED_PEAKS.json does not carry.
//
// crb_probe_fp32_peak: the non-tensor binary32 FMA rate of THIS device at ITS current clocks, measured by a
// kernel that does nothing else (8 independent FFMA chains per thread, 32 resident warps per SM, operands in
// registers).  It is the denominator of the MPC / LQR roofline fractions in bench.py ("fp32 peak, measured in
// the same run"), instead of the nominal SMs x 128 lanes x 2 x clock.
#include "crb_common.cuh"

__global__ void __launch_bounds__(256, 4) crb_probe_ffma_kernel(float* out, int iters, float a, float b) {
  float v0 = threadIdx.x * 1.0e-3f, v1 = v0 + 1.0f, v2 = v0 + 2.0f, v3 = v0 + 3.0f;
  float v4 = v0 + 4.0f, v5 = v0 + 5.0f, v6 = v0 + 6.0f, v7 = v0 + 7.0f;
#pragma unroll 1
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      v0 = fmaf(v0, a, b); v1 = fmaf(v1, a, b); v2 = fmaf(v2, a, b); v3 = fmaf(v3, a, b);
      v4 = fmaf(v4, a, b); v5 = fmaf(v5, a, b); v6 = fmaf(v6, a, b); v7 = fmaf(v7, a, b);
    }
  }
  const float s = ((v0 + v1) + (v2 + v3)) + ((v4 + v5) + (v6 + v7));
  if (s == 123.456f) out[blockIdx.x * blockDim.x + threadIdx.x] = s;  // never true: keeps the chains alive
}

extern "C" int crb_probe_fp32_peak(crb_ctx* ctx, double* tflops_out) {
  CRB_REQUIRE(ctx != nullptr && tflops_out != nullptr, "NULL argument");
  CRB_DEVICE_GUARD(ctx);
  int rc = crb_ctx_scratch_reserve(ctx, (size_t)ctx->sm_count * 8 * 256 * sizeof(float));
  if (rc) return rc;
  const int grid = ctx->sm_count * 8, iters = 4096;   // ~0.3 ms per launch
  float* out = (float*)ctx->scratch;
  cudaStream_t st = ctx->stream;
  for (int w = 0; w < 2; ++w) crb_probe_ffma_kernel<<<grid, 256, 0, st>>>(out, iters, 0.999f, 1.0e-3f);
  double best = 0.0;
  for (int r = 0; r < 5; ++r) {
    CRB_CUDA(cudaEventRecord(ctx->ev_start, st));
    crb_probe_ffma_kernel<<<grid, 256, 0, st>>>(out, iters, 0.999f, 1.0e-3f);
    CRB_CUDA(cudaEventRecord(ctx->ev_stop, st));
    CRB_CUDA(cudaEventSynchronize(ctx->ev_stop));
    float ms = 0.0f;
    CRB_CUDA(cudaEventElapsedTime(&ms, ctx->ev_start, ctx->ev_stop));
    const double flops = 2.0 * 8.0 * 16.0 * (double)iters * (double)grid * 256.0;
    const double tf = flops / ((double)ms * 1.0e-3) / 1.0e12;
    if (tf > best) best = tf;
  }
  CRB_CUDA(cudaGetLastError());
  ctx->launches += 7;
  *tflops_out = best;
  return CRB_OK;
}

// crb_probe_ekf_pattern: the access pattern of the EKF step's default form (crb_ekf_step_kernel<128, 4, 2> in
// crb_ekf.cu: two agents per thread, 8-byte streaming loads and stores of the same 24 / 20 SoA fields, PDL, same
// launch shape) with trivial arithmetic, the ceiling for that pattern (scripts/ekf_ceiling.py).  Every state
// field gets (z0 + z1) + (u0 + u1) of its agent added, in place.
__global__ void __launch_bounds__(128, 4)
crb_probe_ekf_pattern_kernel(int64_t count, float* __restrict__ x, float* __restrict__ P,
                             const float* __restrict__ z, const float* __restrict__ u) {
  const int64_t i = 2 * ((int64_t)blockIdx.x * blockDim.x + threadIdx.x);
  if (i >= count) return;
  const int64_t ld = count;
  crb_pdl_launch_dependents();
  crb_pdl_wait();
  float2 xs[4], Ps[16];
#pragma unroll
  for (int f = 0; f < 4; ++f) xs[f] = __ldcs(reinterpret_cast<const float2*>(x + f * ld + i));
#pragma unroll
  for (int f = 0; f < 16; ++f) Ps[f] = __ldcs(reinterpret_cast<const float2*>(P + f * ld + i));
  const float2 z0 = __ldcs(reinterpret_cast<const float2*>(z + i));
  const float2 z1 = __ldcs(reinterpret_cast<const float2*>(z + ld + i));
  const float2 u0 = __ldcs(reinterpret_cast<const float2*>(u + i));
  const float2 u1 = __ldcs(reinterpret_cast<const float2*>(u + ld + i));
  const float sx = (z0.x + z1.x) + (u0.x + u1.x), sy = (z0.y + z1.y) + (u0.y + u1.y);
#pragma unroll
  for (int f = 0; f < 4; ++f)
    __stcs(reinterpret_cast<float2*>(x + f * ld + i), make_float2(xs[f].x + sx, xs[f].y + sy));
#pragma unroll
  for (int f = 0; f < 16; ++f)
    __stcs(reinterpret_cast<float2*>(P + f * ld + i), make_float2(Ps[f].x + sx, Ps[f].y + sy));
}

extern "C" int crb_probe_ekf_pattern(crb_ctx* ctx, int64_t n, float* x, float* P, const float* z,
                                     const float* u) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_DEVICE_GUARD(ctx);
  CRB_REQUIRE(n >= 0 && n % 2 == 0, "n < 0 or odd");
  if (n == 0) return CRB_OK;
  CRB_REQUIRE(x && P && z && u, "NULL array");
  CRB_REQUIRE((((uintptr_t)x | (uintptr_t)P | (uintptr_t)z | (uintptr_t)u) & 7) == 0,
              "arrays not 8-byte aligned");
  CRB_CUDA(crb_launch_pdl(crb_probe_ekf_pattern_kernel, (unsigned)crb_grid_for(n / 2, 128), 128u, ctx->stream, n,
                          x, P, z, u));
  ctx->launches++;
  return CRB_OK;
}
