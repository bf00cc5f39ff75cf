// crb_common.cuh — context object, error plumbing and launch helpers shared by the libcrb TUs.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/crb.h"

#define CRB_N_PIPE 8  // host-pointer entry points pipeline chunks over this many streams

struct crb_ctx {
  int device;
  int sm_count;
  cudaStream_t own_stream;
  cudaStream_t stream;  // the stream kernels are enqueued on (own_stream or caller's)
  int64_t launches;
  cudaEvent_t ev_start, ev_stop;
  // staging for the *_host entry points: one arena per pipeline slot, grown on demand
  cudaStream_t pipe_stream[CRB_N_PIPE];
  void* pipe_buf[CRB_N_PIPE];
  size_t pipe_cap[CRB_N_PIPE];
  // scratch for reductions / solver workspaces, grown on demand
  void* scratch;
  size_t scratch_cap;
  // MPC solver workspace (two trajectory buffers + gains per problem) for the device-pointer entry
  void* mpc_ws;
  size_t mpc_ws_cap;
  void* host_scratch;  // small pinned buffer for reduction results
  // per-device function attributes already set for this context's device (a second context on another
  // device in the same process must set them again, so these are not process-global latches)
  int mpc_tasks_attr_set;
  int ekf_tma_attr_set;
  int pf_step_attr_set;   // shared-memory carve-out preference of the crb_pf_step kernels (per device)
  int mpc_v0_attr_set;
  unsigned* tickets;      // 64 zeroed words of device memory: "last block finishes the job" counters (kept at zero)
  // NCCL communicator (crb_comm.cu); NULL = single GPU
  void* comm;
  int comm_world, comm_rank;
};

// Makes ctx->device current for the duration of an entry point and restores the caller's device afterwards:
// a process may hold contexts on several devices (one host thread each), and the caller's (torch's) current
// device must not change under it.
struct CrbDeviceGuard {
  int prev;
  bool ok;
  explicit CrbDeviceGuard(const crb_ctx* ctx) : prev(-1), ok(true) {
    if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; cudaGetLastError(); }
    if (prev != ctx->device) ok = cudaSetDevice(ctx->device) == cudaSuccess;
    else prev = -1;
  }
  ~CrbDeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};
#define CRB_DEVICE_GUARD(ctx)                                            \
  CrbDeviceGuard crb_guard_(ctx);                                        \
  if (!crb_guard_.ok) {                                                  \
    crb_set_error("%s: cudaSetDevice(%d) failed", __func__, (ctx)->device); \
    return CRB_ERR_CUDA;                                                 \
  }

void crb_set_error(const char* fmt, ...);

#define CRB_CUDA(call)                                                                      \
  do {                                                                                      \
    cudaError_t e_ = (call);                                                                \
    if (e_ != cudaSuccess) {                                                                \
      crb_set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_));   \
      return e_ == cudaErrorMemoryAllocation ? CRB_ERR_ALLOC : CRB_ERR_CUDA;                \
    }                                                                                       \
  } while (0)

#define CRB_REQUIRE(cond, msg)                                  \
  do {                                                          \
    if (!(cond)) {                                              \
      crb_set_error("%s: invalid argument: %s", __func__, msg); \
      return CRB_ERR_INVALID_ARG;                               \
    }                                                           \
  } while (0)

// Grow-only arenas.
int crb_ctx_pipe_reserve(crb_ctx* ctx, int slot, size_t bytes);
int crb_ctx_scratch_reserve(crb_ctx* ctx, size_t bytes);
int crb_ctx_mpc_ws_reserve(crb_ctx* ctx, size_t bytes);
extern "C" int crb_comm_destroy(crb_ctx* ctx);
extern "C" int crb_comm_allreduce_sum_f64(crb_ctx* ctx, double* buf_dev, int64_t count);

// Strided host<->device block copy for the *_host pipelines: one cudaMemcpy2DAsync per array.  Splitting it
// into per-row 1-D copies makes the pipeline enqueue-bound (scripts/pcie_probe.py compares the two).
static inline cudaError_t crb_copy_rows(void* dst, size_t dpitch, const void* src, size_t spitch,
                                        size_t width, size_t rows, cudaMemcpyKind kind, cudaStream_t st) {
  return cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, rows, kind, st);
}

// Zero-copy eligibility for the *_host entries: a host pointer that the driver reports as pinned AND
// mapped into this device's address space (cudaHostAlloc / cudaMallocHost / crb_host_alloc, or
// cudaHostRegister'ed memory) can be dereferenced by a kernel directly, so the resident kernel is launched
// on it and its coalesced 128-byte loads/stores ride PCIe in both directions at once with no staging
// copy (scripts/zerocopy_probe.py compares it with the staged pipeline).  Pageable pointers return false and
// take the staged pipeline.  CRB_HOST_ZEROCOPY=0
// forces the staged pipeline (A/B, tests).  NULL counts as mappable (optional arrays).
static inline bool crb_zero_copy_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("CRB_HOST_ZEROCOPY");
    on = (e && atoi(e) == 0) ? 0 : 1;
  }
  return on != 0;
}
template <typename T>
static inline bool crb_host_mapped(T* host, T** dev) {
  *dev = nullptr;
  if (host == nullptr) return true;
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, (const void*)host) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  if (at.type != cudaMemoryTypeHost || at.devicePointer == nullptr) return false;
  *dev = (T*)at.devicePointer;
  return true;
}

// Programmatic dependent launch (PDL): back-to-back launches of the short streaming kernels (EKF step, PF
// step: tens of microseconds) otherwise pay the drain of kernel N plus the launch and prologue of kernel N+1
// on every launch.  With the launch attribute below, kernel N+1's CTAs are scheduled as soon as every CTA of
// kernel N has executed crb_pdl_launch_dependents() (or exited); they run their address arithmetic and
// then block in crb_pdl_wait() until kernel N has completed and its writes are visible, so a truly
// dependent sequence (EKF step k+1 reading step k's state) stays correct.  Both instructions are no-ops in
// a kernel launched without the attribute.  CRB_PDL=0 disables the attribute (A/B).
__device__ __forceinline__ void crb_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void crb_pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
static inline bool crb_pdl_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("CRB_PDL");
    on = (e && atoi(e) == 0) ? 0 : 1;
  }
  return on != 0;
}
template <typename... KArgs, typename... Args>
static inline cudaError_t crb_launch_pdl(void (*kernel)(KArgs...), unsigned grid, unsigned block,
                                         cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(block);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = crb_pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

static inline int crb_grid_for(int64_t n, int block) { return (int)((n + block - 1) / block); }

// Streaming (evict-first) global accesses for data that is touched exactly once per launch.
__device__ __forceinline__ float ld_stream(const float* p) { return __ldcs(p); }
__device__ __forceinline__ void st_stream(float* p, float v) { __stcs(p, v); }

// ---- sin/cos with the HOST libm's bits ------------------------------------------------------------------
// The reference calls std::sin / std::cos on floats (src/extended_kalman_filter.cpp:29-33,41-45,
// src/particle_filter.cpp:33-37, src/model_predictive_control.cpp:73-74), i.e. glibc's sinf / cosf.  Those
// are specified only to ~1 ulp, and one ulp of a predicted position is 3e-5 of a particle weight
// (exp(-dz^2 / 2 sigma^2) with sigma = 0.1 m and ranges of ~15 m), so CUDA's own sincosf (also <= 2 ulp, but
// different ulps) cannot meet a per-particle 1e-5 gate on the weights.  glibc >= 2.28 computes sinf / cosf
// in BINARY64: x = (double)y, one multiply-subtract range reduction by pi/2 (exact to 33 bits for |y| < 120),
// a degree-7/8 polynomial, one final rounding to float (sysdeps/ieee754/flt-32/s_sinf.c, s_cosf.c,
// sincosf.h, s_sincosf_data.c).  On x86-64 hosts with FMA (every server CPU of the last decade) glibc's ifunc
// picks the build of those files compiled with -mfma, in which each a + b * c of the source is ONE fused
// operation: that is what is restated here with explicit fma(), operation for operation, and the GPU's FP64
// pipe (IEEE DFMA / DMUL) reproduces it bit for bit.  Checked against the host libm on 3.2e8 floats in
// |y| < 120 (oracle/crb_oracle.c:crb_oracle_libm_sincosf, tests/test_oracle_ekf.py): sin AND cos identical on
// every one of them.  (On a host without FMA, glibc's plain build differs from this on 2e-8 of the inputs, by
// one ulp.)  |y| >= 120 (glibc's table-driven reduce_large) is not restated: CUDA's sincosf is used there (no
// BASELINE workload comes near it).  17 FP64 operations + 3 conversions per call.
static __device__ __noinline__ float2 crb_sincosf_large(float y) {  // by value: no address-taken locals at the call site
  float s, c;
  sincosf(y, &s, &c);
  return make_float2(s, c);
}
// x with the sign flipped when neg != 0 (x * -1.0 without occupying the FP64 pipe)
__device__ __forceinline__ double crb_flip(double x, int neg) {
  return __hiloint2double(__double2hiint(x) ^ (neg ? (int)0x80000000 : 0), __double2loint(x));
}
__device__ __forceinline__ void crb_sincosf_libm(float y, float& sn, float& cs) {
  const unsigned top = (__float_as_uint(y) >> 20) & 0x7ffu;
  if (top >= 0x42fu) {  // |y| >= 120, inf, nan: out of line (CUDA's Payne-Hanek path is long)
    const float2 sc = crb_sincosf_large(y);
    sn = sc.x;
    cs = sc.y;
    return;
  }
  double x = (double)y;
  int n = 0;
  if (top >= 0x3f4u) {  // |y| >= pi/4 (abstop12(0x1.921FB6p-1f) = 0x3f4): reduce_fast
    const double r = x * 0x1.45F306DC9C883p+23;
    n = ((int)r + 0x800000) >> 24;
    x = fma(-(double)n, 0x1.921FB54442D18p0, x);
  } else if (top < 0x398u) {  // |y| < 2^-12
    sn = y;
    cs = 1.0f;
    return;
  }
  const double x2 = x * x;
  const int neg_s = (n + 1) & 2;  // sign[n & 3] = {1, -1, -1, 1}
  const int neg_c = n & 2;        // second table entry: cosine coefficients negated
  const double xs = crb_flip(x, neg_s);
  // sine polynomial on xs (its coefficients are the same in both table entries)
  const double x3 = xs * x2;
  const double s1 = fma(x2, -0x1.994eb3774cf24p-13, 0x1.1107605230bc4p-7);
  const double x7 = x3 * x2;
  const double sp = fma(x3, -0x1.555545995a603p-3, xs);
  const float ps = (float)fma(x7, s1, sp);
  // cosine polynomial: negating all five coefficients negates every intermediate and the result exactly, so
  // the polynomial is evaluated with the first table entry and the sign applied to the rounded float
  const double x4 = x2 * x2;
  const double c2 = fma(x2, 0x1.99343027bf8c3p-16, -0x1.6c087e89a359dp-10);
  const double c1 = fma(x2, -0x1.ffffffd0c621cp-2, 1.0);
  const double x6 = x4 * x2;
  const double cp = fma(x4, 0x1.55553e1068f19p-5, c1);
  const float pc0 = (float)fma(x6, c2, cp);
  const float pc = __int_as_float(__float_as_int(pc0) ^ (neg_c ? (int)0x80000000 : 0));
  // sinf uses the sine polynomial for even n, cosf for odd n (and vice versa)
  sn = (n & 1) ? pc : ps;
  cs = (n & 1) ? ps : pc;
}

// ---- tanf with the HOST libm's bits ---------------------------------------------------------------------
// The reference calls std::tan on a float (include/motion_model.h:105), i.e. glibc's tanf.  glibc 2.39 computes
// it with fdlibm's binary32 s_tanf.c / k_tanf.c (Sun Microsystems, freely redistributable): |x| <= pi/4 goes
// straight to __kernel_tanf(x, 0, 1); above that, __ieee754_rem_pio2f reduces by pi/2 with the same binary64
// reduce_fast as sinf (n from the 2^24/pi product, then x - n * pi/2 as a separate multiply and subtract: unlike
// sinf's, this file is not built with FMA) and splits the remainder into y0 = (float)r, y1 = (float)(r - y0);
// __kernel_tanf(y0, y1, +-1) then works in float only.  Restated operation for operation with explicitly rounded
// intrinsics, so it does not depend on the TU's -fmad setting.  Checked against the host tanf on every one of the
// 2,246,049,792 floats with |x| < 120 (oracle/crb_oracle_mptg.c: crb_oracle_libm_tanf_census, tests/test_mptg.py).
// |x| >= 120 (glibc's reduce_large) is not restated: crb_tanf_libm_in_range() says whether x is inside the
// proven range, and callers must not use the result outside it.  Inf and NaN give NaN, as glibc does.
__device__ __forceinline__ bool crb_tanf_libm_in_range(float x) {
  const unsigned ix = __float_as_uint(x) & 0x7fffffffu;
  return ix < 0x42f00000u || ix >= 0x7f800000u;  // |x| < 120, or not finite
}
static __device__ __noinline__ float crb_tanf_kernel(float x, float y, int iy) {  // __kernel_tanf, iy = +1 / -1
  const float pio4 = 7.8539812565e-01f, pio4lo = 3.7748947079e-08f;
  const float T0 = 3.3333334327e-01f, T1 = 1.3333334029e-01f, T2 = 5.3968254477e-02f, T3 = 2.1869488060e-02f,
              T4 = 8.8632395491e-03f, T5 = 3.5920790397e-03f, T6 = 1.4562094584e-03f, T7 = 5.8804126456e-04f,
              T8 = 2.4646313977e-04f, T9 = 7.8179444245e-05f, T10 = 7.1407252108e-05f, T11 = -1.8558637748e-05f,
              T12 = 2.5907305826e-05f;
  const int hx = __float_as_int(x);
  const int ix = hx & 0x7fffffff;
  if (ix < 0x39000000) {  // |x| < 2^-13
    if (iy == 1) return x;
    if (ix == 0) return __fdiv_rn(1.0f, fabsf(x));  // glibc's one / fabsf(x) for x = +-0, iy = -1
    return __fdiv_rn(-1.0f, x);
  }
  const bool big = ix >= 0x3f2ca140;  // |x| >= 0.6744
  if (big) {
    if (hx < 0) {
      x = -x;
      y = -y;
    }
    const float z = __fsub_rn(pio4, x), w = __fsub_rn(pio4lo, y);
    x = __fadd_rn(z, w);
    y = 0.0f;
    if (fabsf(x) < 0x1p-13f) {  // (1 - ((hx >> 30) & 2)) * iy * (1.0f - 2 * iy * x): products by +-1, +-2 are exact
      const float sg = (float)((1 - ((hx >> 30) & 2)) * iy);
      return __fmul_rn(sg, __fsub_rn(1.0f, __fmul_rn((float)(2 * iy), x)));
    }
  }
  const float z = __fmul_rn(x, x);
  const float w = __fmul_rn(z, z);
  float r = __fadd_rn(T1, __fmul_rn(w, __fadd_rn(T3, __fmul_rn(w, __fadd_rn(T5, __fmul_rn(w, __fadd_rn(T7,
            __fmul_rn(w, __fadd_rn(T9, __fmul_rn(w, T11))))))))));
  float v = __fmul_rn(z, __fadd_rn(T2, __fmul_rn(w, __fadd_rn(T4, __fmul_rn(w, __fadd_rn(T6, __fmul_rn(w,
            __fadd_rn(T8, __fmul_rn(w, __fadd_rn(T10, __fmul_rn(w, T12)))))))))));
  const float s = __fmul_rn(z, x);
  r = __fadd_rn(y, __fmul_rn(z, __fadd_rn(__fmul_rn(s, __fadd_rn(r, v)), y)));
  r = __fadd_rn(r, __fmul_rn(T0, s));
  const float ww = __fadd_rn(x, r);
  if (big) {
    const float fv = (float)iy;
    const float q = __fsub_rn(__fdiv_rn(__fmul_rn(ww, ww), __fadd_rn(ww, fv)), r);
    return __fmul_rn((float)(1 - ((hx >> 30) & 2)), __fsub_rn(fv, __fmul_rn(2.0f, __fsub_rn(x, q))));
  }
  if (iy == 1) return ww;
  // -1 / (x + r) to full precision
  const float zz = __int_as_float(__float_as_int(ww) & (int)0xfffff000);
  const float vv = __fsub_rn(r, __fsub_rn(zz, x));
  const float a = __fdiv_rn(-1.0f, ww);
  const float t = __int_as_float(__float_as_int(a) & (int)0xfffff000);
  const float ss = __fadd_rn(1.0f, __fmul_rn(t, zz));
  return __fadd_rn(t, __fmul_rn(a, __fadd_rn(ss, __fmul_rn(t, vv))));
}
__device__ __forceinline__ float crb_tanf_libm(float x) {
  const unsigned ix = __float_as_uint(x) & 0x7fffffffu;
  if (ix <= 0x3f490fdau) return crb_tanf_kernel(x, 0.0f, 1);  // |x| <= pi/4
  if (ix >= 0x7f800000u) return __fsub_rn(x, x);             // inf, NaN
  // reduce_fast (|x| < 120; larger x gets no meaningful result, see crb_tanf_libm_in_range)
  const double dx = (double)x;
  const int n = ((int)__dmul_rn(dx, 0x1.45F306DC9C883p+23) + 0x800000) >> 24;
  const double d = __dsub_rn(dx, __dmul_rn((double)n, 0x1.921FB54442D18p0));
  const float y0 = __double2float_rn(d);
  const float y1 = __double2float_rn(__dsub_rn(d, (double)y0));
  return crb_tanf_kernel(y0, y1, 1 - ((n & 1) << 1));
}
