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
  // grid planner workspace (query counter + one search slot per lane, crb_grid.cu), grown on demand
  void* grid_ws;
  size_t grid_ws_cap;
  void* rrt_counter;  // RRT query counter (crb_rrt.cu), allocated on first use
  void* host_scratch;  // small pinned buffer for reduction results
  // per-device function attributes already set for this context's device (a second context on another
  // device in the same process must set them again, so these are not process-global latches)
  int mpc_tasks_attr_set;
  int pf_step_attr_set;   // shared-memory carve-out preference of the crb_pf_step kernels (per device)
  int mpc_v0_attr_set;
  int pf_fleet_attr_set;  // crb_pf_fleet_kernel's dynamic shared-memory limit raised to FLEET_SMEM_MAX
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
// CRB_OK, or CRB_ERR_NO_DEVICE and the error string "<fn>: no usable CUDA device; ..." without a usable CUDA device:
// an entry point calls it after validating its arguments, as there is no CPU fallback.
int crb_require_device(const char* fn);

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

// The obstacle list of agent i in an obstacle store (crb.h): rows [b, e) of ob, checked before any row is read.
// ob_of NULL means one list, [0, n_rows), for every agent (a shared-list entry point, whose n_rows the host checked).
// Otherwise ob_of[i] must lie in [0, n_sets) and 0 <= ob_off[s] <= ob_off[s + 1] <= n_rows with at most cap rows;
// false for a reference that fails (b = e = 0 then).  Empty lists are valid.
__device__ __forceinline__ bool crb_obstacle_list(int64_t i, const int64_t* __restrict__ ob_off, int32_t n_sets,
                                                  const int32_t* __restrict__ ob_of, int64_t n_rows, int64_t cap,
                                                  int64_t& b, int64_t& e) {
  b = 0;
  e = ob_of ? 0 : n_rows;
  if (!ob_of) return true;
  const int32_t s = ob_of[i];
  if (s < 0 || s >= n_sets) return false;
  const int64_t lo = ob_off[s], hi = ob_off[s + 1];
  if (lo < 0 || lo > hi || hi > n_rows || hi - lo > cap) return false;
  b = lo;
  e = hi;
  return true;
}

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
// pipe (IEEE DFMA / DMUL) reproduces it bit for bit.  |y| >= 120 takes glibc's reduce_large: an exact 2.62
// fixed-point remainder from three 32x32-bit integer products with a window of 2/pi, converted to binary64 and
// scaled by pi/2^62, then the same polynomial; integer and binary64 work only, so it is reproduced bit for bit
// too.  The C restatement (oracle/crb_oracle.c:crb_oracle_libm_sincosf) equals the host libm, sin AND cos, on
// every finite float with |y| >= 120 and on a dense sample below (tests/test_oracle_ekf.py), and this function
// equals the C restatement on all 2^32 bit patterns on the device (tests/test_ekf_edges.py).  (On a host without
// FMA, glibc's plain build differs from this on 2e-8 of the inputs, by one ulp.)  Inf and NaN give NaN.  17 FP64
// operations + 3 conversions per call below 120.
// x with the sign flipped when neg != 0 (x * -1.0 without occupying the FP64 pipe)
__device__ __forceinline__ double crb_flip(double x, int neg) {
  return __hiloint2double(__double2hiint(x) ^ (neg ? (int)0x80000000 : 0), __double2loint(x));
}
// sinf_poly for both results on the reduced argument x (|x| <= pi/4): m picks the signs (sign table and the
// negated cosine table), n the polynomial (sinf takes the sine polynomial for even n, cosf for odd n)
__device__ __forceinline__ void crb_sincosf_poly(double x, int n, int m, float& sn, float& cs) {
  const double x2 = x * x;
  const int neg_s = (m + 1) & 2;  // sign[m & 3] = {1, -1, -1, 1}
  const int neg_c = m & 2;        // second table entry: cosine coefficients negated
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
// 2/pi in 8-bit steps (glibc's __inv_pio4): word k holds bits [8k - 24, 8k + 8) of its binary fraction
static __device__ __constant__ const uint32_t crb_inv_pio4[24] = {
    0xa2,       0xa2f9,     0xa2f983,   0xa2f9836e, 0xf9836e4e, 0x836e4e44, 0x6e4e4415, 0x4e441529,
    0x441529fc, 0x1529fc27, 0x29fc2757, 0xfc2757d1, 0x2757d1f5, 0x57d1f534, 0xd1f534dd, 0xf534ddc0,
    0x34ddc0db, 0xddc0db62, 0xc0db6295, 0xdb629599, 0x6295993c, 0x95993c43, 0x993c4390, 0x3c439041};
// glibc's reduce_large for |y| >= 120, out of line so that the hot paths (whose arguments stay far below 120) keep
// their registers: |y| = (n + r / 2^62) * pi/2 in exact 2.62 fixed point from the 24-bit significand and a 96-bit
// window of 2/pi chosen by the exponent.  Returns r * pi/2^62 (|.| <= pi/4) with n in .y's low word and the sign
// quadrant n + signbit(y) in its high word; inf and nan return y - y (nan), which the polynomial passes on.
static __device__ __noinline__ double2 crb_sincosf_reduce_large(float y) {  // by value: no address-taken locals
  uint32_t xi = __float_as_uint(y);
  if ((xi & 0x7fffffffu) >= 0x7f800000u) return make_double2((double)__fsub_rn(y, y), 0.0);
  const uint32_t* arr = &crb_inv_pio4[(xi >> 26) & 15];
  const int sign = (int)(xi >> 31);
  xi = ((xi & 0xffffffu) | 0x800000u) << ((xi >> 23) & 7);
  uint64_t res0 = (uint64_t)(xi * arr[0]);  // only the low 32 bits of the top product matter
  const uint64_t res1 = (uint64_t)xi * arr[4];
  const uint64_t res2 = (uint64_t)xi * arr[8];
  res0 = ((res2 >> 32) | (res0 << 32)) + res1;
  const uint64_t n = (res0 + (1ull << 61)) >> 62;
  res0 -= n << 62;
  const double x = __dmul_rn(__ll2double_rn((long long)res0), 0x1.921FB54442D18p-62);
  return make_double2(x, __hiloint2double((int)n + sign, (int)n));
}
__device__ __forceinline__ void crb_sincosf_libm(float y, float& sn, float& cs) {
  const unsigned top = (__float_as_uint(y) >> 20) & 0x7ffu;
  double x = (double)y;
  int n = 0, m;
  if (top >= 0x42fu) {  // |y| >= 120, inf, nan
    const double2 r = crb_sincosf_reduce_large(y);
    x = r.x;
    n = __double2loint(r.y);
    m = __double2hiint(r.y);
  } else {
    if (top >= 0x3f4u) {  // |y| >= pi/4 (abstop12(0x1.921FB6p-1f) = 0x3f4): reduce_fast
      const double r = x * 0x1.45F306DC9C883p+23;
      n = ((int)r + 0x800000) >> 24;
      x = fma(-(double)n, 0x1.921FB54442D18p0, x);
    } else if (top < 0x398u) {  // |y| < 2^-12
      sn = y;
      cs = 1.0f;
      return;
    }
    m = n;
  }
  crb_sincosf_poly(x, n, m, sn, cs);
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

// ---- atan2f with the HOST libm's bits -------------------------------------------------------------------
// The reference calls std::atan2 on floats (include/rrt.h:113), i.e. glibc's atan2f.  glibc 2.39 computes it with
// fdlibm's binary32 e_atan2f.c on top of __atanf (s_atanf.c) (Sun Microsystems, freely redistributable), in float
// only; it is not (float)atan2((double)y, (double)x).  Restated operation for operation with explicitly rounded
// intrinsics, so it does not depend on the TU's -fmad setting.  The C twin (oracle/crb_oracle_rrt.c) equals the host
// atanf on every non-negative float and the host atan2f on dense pairs and every sign / zero / inf / NaN case
// (tests/test_rrt.py); this equals the C twin on the device.
static __device__ __noinline__ float crb_atanf_libm(float x) {  // __atanf
  const int hx = __float_as_int(x);
  const int ix = hx & 0x7fffffff;
  int id;
  if (ix >= 0x4c000000) {  // |x| >= 2^25
    if (ix > 0x7f800000) return __fadd_rn(x, x);
    return hx > 0 ? __fadd_rn(1.5707962513e+00f, 7.5497894159e-08f) : __fsub_rn(-1.5707962513e+00f, 7.5497894159e-08f);
  }
  if (ix < 0x3ee00000) {              // |x| < 0.4375
    if (ix < 0x31000000) return x;    // |x| < 2^-29
    id = -1;
  } else {
    x = fabsf(x);
    if (ix < 0x3f980000) {      // |x| < 1.1875
      if (ix < 0x3f300000) {    // 7/16 <= |x| < 11/16
        id = 0;
        x = __fdiv_rn(__fsub_rn(__fmul_rn(2.0f, x), 1.0f), __fadd_rn(2.0f, x));
      } else {                  // 11/16 <= |x| < 19/16
        id = 1;
        x = __fdiv_rn(__fsub_rn(x, 1.0f), __fadd_rn(x, 1.0f));
      }
    } else if (ix < 0x401c0000) {  // |x| < 2.4375
      id = 2;
      x = __fdiv_rn(__fsub_rn(x, 1.5f), __fadd_rn(1.0f, __fmul_rn(1.5f, x)));
    } else {                       // 2.4375 <= |x| < 2^25
      id = 3;
      x = __fdiv_rn(-1.0f, x);
    }
  }
  const float z = __fmul_rn(x, x);
  const float w = __fmul_rn(z, z);
  const float s1 = __fmul_rn(z, __fadd_rn(3.3333334327e-01f, __fmul_rn(w, __fadd_rn(1.4285714924e-01f,
                   __fmul_rn(w, __fadd_rn(9.0908870101e-02f, __fmul_rn(w, __fadd_rn(6.6610731184e-02f,
                   __fmul_rn(w, __fadd_rn(4.9768779427e-02f, __fmul_rn(w, 1.6285819933e-02f)))))))))));
  const float s2 = __fmul_rn(w, __fadd_rn(-2.0000000298e-01f, __fmul_rn(w, __fadd_rn(-1.1111110449e-01f,
                   __fmul_rn(w, __fadd_rn(-7.6918758452e-02f, __fmul_rn(w, __fadd_rn(-5.8335702866e-02f,
                   __fmul_rn(w, -3.6531571299e-02f)))))))));
  if (id < 0) return __fsub_rn(x, __fmul_rn(x, __fadd_rn(s1, s2)));
  // atanhi[id], atanlo[id] (selects, not an indexed array: no local memory)
  const float hi = id == 0 ? 4.6364760399e-01f : id == 1 ? 7.8539812565e-01f : id == 2 ? 9.8279368877e-01f
                                                                                       : 1.5707962513e+00f;
  const float lo = id == 0 ? 5.0121582440e-09f : id == 1 ? 3.7748947079e-08f : id == 2 ? 3.4473217170e-08f
                                                                                       : 7.5497894159e-08f;
  const float r = __fsub_rn(hi, __fsub_rn(__fsub_rn(__fmul_rn(x, __fadd_rn(s1, s2)), lo), x));
  return hx < 0 ? -r : r;
}
__device__ __forceinline__ float crb_atan2f_libm(float y, float x) {
  const float tiny = 1.0e-30f, pi_o_4 = 7.8539818525e-01f, pi_o_2 = 1.5707963705e+00f, pi = 3.1415927410e+00f,
              pi_lo = -8.7422776573e-08f;
  const int hx = __float_as_int(x), ix = hx & 0x7fffffff;
  const int hy = __float_as_int(y), iy = hy & 0x7fffffff;
  if (ix > 0x7f800000 || iy > 0x7f800000) return __fadd_rn(x, y);  // NaN
  if (hx == 0x3f800000) return crb_atanf_libm(y);                   // x = 1
  const int m = ((hy >> 31) & 1) | ((hx >> 30) & 2);                 // 2 * sign(x) + sign(y)
  const float pi_t = __fadd_rn(pi, tiny), pi_o_2_t = __fadd_rn(pi_o_2, tiny);
  if (iy == 0) return m < 2 ? y : (m == 2 ? pi_t : __fsub_rn(-pi, tiny));
  if (ix == 0) return hy < 0 ? __fsub_rn(-pi_o_2, tiny) : pi_o_2_t;
  if (ix == 0x7f800000) {
    if (iy == 0x7f800000) {
      const float a = m < 2 ? pi_o_4 : __fmul_rn(3.0f, pi_o_4);
      return (m & 1) ? __fsub_rn(-a, tiny) : __fadd_rn(a, tiny);
    }
    return m == 0 ? 0.0f : m == 1 ? -0.0f : m == 2 ? pi_t : __fsub_rn(-pi, tiny);
  }
  if (iy == 0x7f800000) return hy < 0 ? __fsub_rn(-pi_o_2, tiny) : pi_o_2_t;
  const int k = (iy - ix) >> 23;
  float z;
  if (k > 60) z = __fadd_rn(pi_o_2, __fmul_rn(0.5f, pi_lo));  // |y / x| > 2^60
  else if (hx < 0 && k < -60) z = 0.0f;                       // |y| / x < -2^60
  else z = crb_atanf_libm(fabsf(__fdiv_rn(y, x)));
  switch (m) {
    case 0: return z;
    case 1: return -z;
    case 2: return __fsub_rn(pi, __fsub_rn(z, pi_lo));
    default: return __fsub_rn(__fsub_rn(z, pi_lo), pi);
  }
}

// ---- YAW_P2P with the reference's bits --------------------------------------------------------------------
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

// ---- (float)atan2(y, 1.0) with the HOST libm's bits (DESIGN.md §3.4) ----------------------------------------
// The LQR programs' feed-forward is float ff = std::atan2(L*k, (double)1.0) (src/lqr_steer_control.cpp:125,
// src/lqr_speed_steer_control.cpp:142): glibc's binary64 atan2 narrowed to float.  The narrowing is what has to be
// reproduced, and it only depends on the binary64 result where that result lies within a few binary64 ulps of a
// float rounding midpoint.  Fast path: CUDA's atan (<= 2 ulp) and glibc's (<= 1 ulp) are both within 3 ulps of the
// true value's neighbourhood, so when the binary64 values 4 ulps either side of CUDA's result narrow to the same
// float, that float is glibc's too.  Otherwise atan(y) is evaluated in double-double (relative error ~2^-100) and
// its correctly rounded binary64 head is narrowed: glibc is correctly rounded wherever that matters, which the census
// over every non-negative float k with y = 0.5 * k checks (tests/test_lqr_track.py).  Odd in y, as glibc is.
struct crb_dd { double hi, lo; };
__device__ __forceinline__ crb_dd crb_dd_fast(double a, double b) {  // |a| >= |b|
  const double s = __dadd_rn(a, b);
  return {s, __dsub_rn(b, __dsub_rn(s, a))};
}
__device__ __forceinline__ crb_dd crb_dd_add(crb_dd a, crb_dd b) {
  const double s = __dadd_rn(a.hi, b.hi);
  const double bb = __dsub_rn(s, a.hi);
  const double e = __dadd_rn(__dsub_rn(a.hi, __dsub_rn(s, bb)), __dsub_rn(b.hi, bb));
  return crb_dd_fast(s, __dadd_rn(e, __dadd_rn(a.lo, b.lo)));
}
__device__ __forceinline__ crb_dd crb_dd_mul(crb_dd a, crb_dd b) {
  const double p = __dmul_rn(a.hi, b.hi);
  const double e = __dadd_rn(__fma_rn(a.hi, b.hi, -p), __dadd_rn(__dmul_rn(a.hi, b.lo), __dmul_rn(a.lo, b.hi)));
  return crb_dd_fast(p, e);
}
__device__ __forceinline__ crb_dd crb_dd_neg(crb_dd a) { return {-a.hi, -a.lo}; }
__device__ __forceinline__ crb_dd crb_dd_div(crb_dd a, crb_dd b) {  // three quotient digits
  const double q1 = __ddiv_rn(a.hi, b.hi);
  const crb_dd r1 = crb_dd_add(a, crb_dd_neg(crb_dd_mul({q1, 0.0}, b)));
  const double q2 = __ddiv_rn(r1.hi, b.hi);
  const crb_dd r2 = crb_dd_add(r1, crb_dd_neg(crb_dd_mul({q2, 0.0}, b)));
  const double q3 = __ddiv_rn(r2.hi, b.hi);
  return crb_dd_add(crb_dd_fast(q1, q2), {q3, 0.0});
}
// atan(y) for finite y >= 0: atan(x) = atan(j/8) + atan(t), t = (x - j/8) / (1 + x j/8), |t| <= 1/16, with x = y or
// 1/y (then pi/2 minus the result); the series in t^2 to t^25 (truncation < 2^-100 relative).  Out of line: it is
// the rare path.
static __device__ __noinline__ crb_dd crb_atan_dd(double y) {
  const bool inv = y > 1.0;
  crb_dd x = {y, 0.0};
  if (inv) {
    const double h = __drcp_rn(y);
    x = crb_dd_fast(h, __ddiv_rn(__fma_rn(-h, y, 1.0), y));
  }
  const int j = (int)__dadd_rn(__dmul_rn(x.hi, 8.0), 0.5);
  const double c = __dmul_rn((double)j, 0.125);
  // atan(j/8), j = 0..8, as double-double (selects, not an indexed array: no local memory)
  const double ah = j == 0 ? 0.0 : j == 1 ? 0x1.fd5ba9aac2f6ep-4 : j == 2 ? 0x1.f5b75f92c80ddp-3
                  : j == 3 ? 0x1.6f61941e4def1p-2 : j == 4 ? 0x1.dac670561bb4fp-2 : j == 5 ? 0x1.1e00babdefeb4p-1
                  : j == 6 ? 0x1.4978fa3269ee1p-1 : j == 7 ? 0x1.700a7c5784634p-1 : 0x1.921fb54442d18p-1;
  const double al = j == 0 ? 0.0 : j == 1 ? -0x1.cd37686760c17p-59 : j == 2 ? 0x1.8ab6e3cf7afbdp-57
                  : j == 3 ? -0x1.c63aae6f6e918p-56 : j == 4 ? 0x1.a2b7f222f65e2p-56 : j == 5 ? -0x1.928df287a668fp-58
                  : j == 6 ? 0x1.2419a87f2a458p-56 : j == 7 ? -0x1.8c34d25aadef6p-56 : 0x1.1a62633145c07p-55;
  const crb_dd num = crb_dd_add(x, {-c, 0.0});
  const crb_dd den = crb_dd_add(crb_dd_mul(x, {c, 0.0}), {1.0, 0.0});
  const crb_dd t = crb_dd_div(num, den);
  const crb_dd s = crb_dd_mul(t, t);
  crb_dd q = {__ddiv_rn(1.0, 25.0), 0.0};
  for (int i = 11; i >= 0; --i) {  // q = sum_i (-1)^i t^(2i) / (2i + 1), Horner in s = t^2
    const double dn = (double)(2 * i + 1);
    const double h = __ddiv_rn(1.0, dn);
    crb_dd ci = crb_dd_fast(h, __ddiv_rn(__fma_rn(-h, dn, 1.0), dn));
    if (i & 1) ci = crb_dd_neg(ci);
    q = crb_dd_add(ci, crb_dd_mul(s, q));
  }
  crb_dd r = crb_dd_add({ah, al}, crb_dd_mul(t, q));
  if (inv) r = crb_dd_add({0x1.921fb54442d18p+0, 0x1.1a62633145c07p-54}, crb_dd_neg(r));
  return r;
}
__device__ __forceinline__ float crb_atan2_1_to_float(double y) {
  const double d = atan(y);  // NaN for NaN, +-pi/2 for +-inf
  if (!isfinite(y)) return __double2float_rn(d);
  const double ad = fabs(d);
  const long long b = __double_as_longlong(ad);
  if (__double2float_rn(__longlong_as_double(b > 4 ? b - 4 : 0)) == __double2float_rn(__longlong_as_double(b + 4)))
    return __double2float_rn(d);
  const float f = __double2float_rn(crb_atan_dd(fabs(y)).hi);
  return y < 0.0 ? -f : f;
}
