// crb_slp.cu — the state lattice planner's terminal-state samplers and lookup-table search for a batch of
// queries, for sm_90a.
//
// Replaces calc_uniform_polar_states / calc_biased_polar_states / calc_lane_states (with sample_states) and
// search_nearest_one_from_lookuptable of src/state_lattice_planner.cpp:29-135.  generate_path :137-155 is that
// search followed by crb_mptg_optimize_batched (crb_mptg.cu), which the layers above compose.  Bit-exact with the
// reference compiled for x86-64: every float and double operation is an explicitly rounded intrinsic, so the TU's
// -fmad setting does not matter, every mixed float / double expression keeps the reference's types, and sin / cos
// are glibc's sinf / cosf (crb_sincosf_libm).
//
// Mapping: one thread per query (sampler) or per target (search), all state in registers.  The biased sampler keeps
// no per-thread array: its first pass sums the ns - 1 samples, and its scan recomputes each normalised sample as it
// reaches it and carries the two prefix sums csumnav[p - 1] and csumnav[p] the back-stepping scan can ask for.
#include <float.h>

#include "crb_common.cuh"

#define SLP_BLOCK 128

namespace {

__device__ __forceinline__ float slp_nan() { return __int_as_float(0x7fc00000); }

// a finite argument outside crb_sincosf_libm's proven range (inf and NaN give NaN, as glibc does)
__device__ __forceinline__ bool slp_trig_out_of_range(float a) { return fabsf(a) >= 120.0f && isfinite(a); }

// Output slot k of query i: target [3][n_q * S].
struct Out {
  float* t;
  int64_t ncol, col0;
  __device__ __forceinline__ void put(int k, float x, float y, float yaw) const {
    t[col0 + k] = x;
    t[ncol + col0 + k] = y;
    t[2 * ncol + col0 + k] = yaw;
  }
};

// Per-query floats and shared integers of the polar samplers.
struct Polar {
  float a_min, a_max, p_min, p_max, d;  // d: sample_states' int d, converted once (int * float is a float product)
  int nh;
};

// sample_states :29-45 for one angle sample: nh states at k, k + 1, ...  False (nothing written) when the angle is a
// finite value outside the sin / cos range.
__device__ __forceinline__ bool slp_emit_polar(const Polar& P, float item, const Out& o, int& k) {
  const float a = __fadd_rn(P.a_min, __fmul_rn(__fsub_rn(P.a_max, P.a_min), item));
  if (slp_trig_out_of_range(a)) return false;
  float sn, cs;
  crb_sincosf_libm(a, sn, cs);
  const float xf = __fmul_rn(P.d, cs), yf = __fmul_rn(P.d, sn);
  const float span = __fsub_rn(P.p_max, P.p_min);
  if (P.nh == 1) {  // (p_max - p_min) / 2.0 + a in double (not the midpoint), narrowed by the assignment
    o.put(k++, xf, yf, __double2float_rn(__dadd_rn(__ddiv_rn((double)span, 2.0), (double)a)));
    return true;
  }
  const float den = __int2float_rn(P.nh - 1);
  for (int j = 0; j < P.nh; ++j)  // p_min + (p_max - p_min) * j / (nh - 1) + a, all float
    o.put(k++, xf, yf, __fadd_rn(__fadd_rn(P.p_min, __fdiv_rn(__fmul_rn(span, __int2float_rn(j)), den)), a));
  return true;
}

// calc_uniform_polar_states :47-56: angle sample i is (float)(i * 1.0 / (nxy - 1)), computed in double
__device__ __forceinline__ bool slp_uniform(const Polar& P, int nxy, const Out& o, int& k) {
  const double den = (double)(nxy - 1);
  for (int i = 0; i < nxy; ++i)
    if (!slp_emit_polar(P, __double2float_rn(__ddiv_rn((double)i, den)), o, k)) return false;
  return true;
}

// asi_sample i of calc_biased_polar_states :67 and its cnav_sample :69: M_PI - |asi - goal| with the abs in float,
// the subtraction in double, narrowed to float
__device__ __forceinline__ float slp_cnav(const Polar& P, float goal, float span, float nsm1, int i) {
  const float asi = __fadd_rn(P.a_min, __fdiv_rn(__fmul_rn(span, __int2float_rn(i)), nsm1));
  return __double2float_rn(__dsub_rn(kPi, (double)fabsf(__fsub_rn(asi, goal))));
}

// calc_biased_polar_states :58-99
__device__ __forceinline__ bool slp_biased(const Polar& P, float goal, int ns, int nxy, const Out& o, int& k) {
  const float span = __fsub_rn(P.a_max, P.a_min), nsm1 = __int2float_rn(ns - 1);
  float cmax = FLT_MIN, csum = 0.0f;  // cnav_max starts at numeric_limits<float>::min(), the smallest normal
  for (int i = 0; i < ns - 1; ++i) {
    const float c = slp_cnav(P, goal, span, nsm1, i);
    csum = __fadd_rn(csum, c);
    if (cmax < c) cmax = c;
  }
  const float den = __fsub_rn(__fmul_rn(cmax, __int2float_rn(ns)), csum);  // cnav_max * ns - cnav_sum
  // csumnav[p] = c_cur and csumnav[p - 1] = c_prev.  A match at j leaves p = j and restarts the scan at j - 1, so
  // no scan ever asks for an index below p - 1 (and never for csumnav[-1]: j = -1 gives j / ns < 0 <= i / (nxy-1)).
  int p = -1;
  float c_prev = slp_nan(), c_cur = 0.0f;
  int li = 0;
  const double dns = (double)ns, dnxy = (double)(nxy - 1);
  for (int i = 0; i < nxy; ++i) {
    const double ri = __ddiv_rn((double)i, dnxy);
    for (int j = li; j < ns - 1; ++j) {
      if (__ddiv_rn((double)j, dns) >= ri) {  // j * 1.0 / ns >= i * 1.0 / (nxy - 1), in double
        while (p < j) {
          ++p;
          c_prev = c_cur;
          c_cur = __fadd_rn(c_cur, __fdiv_rn(__fsub_rn(cmax, slp_cnav(P, goal, span, nsm1, p)), den));
        }
        if (!slp_emit_polar(P, j == p ? c_cur : c_prev, o, k)) return false;
        li = j - 1;
        break;
      }
    }
  }
  return true;
}

// calc_lane_states :101-113
__device__ __forceinline__ bool slp_lane(float l_center, float l_heading, float l_width, float v_width, float d,
                                         int nxy, const Out& o, int& k) {
  if (slp_trig_out_of_range(l_heading)) return false;
  float sn, cs;
  crb_sincosf_libm(l_heading, sn, cs);
  const float xc = __fadd_rn(__fmul_rn(cs, d), __fmul_rn(sn, l_center));
  const float yc = __fadd_rn(__fmul_rn(sn, d), __fmul_rn(cs, l_center));  // + cos * l_center, as the reference has it
  const float w = __fsub_rn(l_width, v_width), den = __int2float_rn(nxy - 1);
  const double half = __dmul_rn(-0.5, (double)w);
  for (int i = 0; i < nxy; ++i) {
    // -0.5 * w + w * i / (nxy - 1): the sum and its first term in double, the second term in float
    const float delta = __double2float_rn(__dadd_rn(half, (double)__fdiv_rn(__fmul_rn(w, __int2float_rn(i)), den)));
    o.put(k++, __fsub_rn(xc, __fmul_rn(delta, sn)), __fadd_rn(yc, __fmul_rn(delta, cs)), l_heading);
  }
  return true;
}

}  // namespace

__global__ void __launch_bounds__(SLP_BLOCK)
crb_slp_sample_kernel(int64_t nq, crb_slp_sampler s, int S, const float* __restrict__ qp, float* __restrict__ tgt,
                      int32_t* __restrict__ nst, int32_t* __restrict__ statusp) {
  const int64_t i = (int64_t)blockIdx.x * SLP_BLOCK + threadIdx.x;
  if (i >= nq) return;
  const Out o{tgt, nq * S, i * S};
  int k = 0;
  bool ok;
  if (s.kind == CRB_SLP_LANE) {
    ok = slp_lane(qp[i], qp[nq + i], qp[2 * nq + i], qp[3 * nq + i], qp[4 * nq + i], s.nxy, o, k);
  } else {
    const int f0 = s.kind == CRB_SLP_BIASED ? 1 : 0;
    Polar P;
    P.a_min = qp[(f0 + 0) * nq + i];
    P.a_max = qp[(f0 + 1) * nq + i];
    P.p_min = qp[(f0 + 2) * nq + i];
    P.p_max = qp[(f0 + 3) * nq + i];
    P.d = __int2float_rn(s.d);
    P.nh = s.nh;
    ok = s.kind == CRB_SLP_BIASED ? slp_biased(P, qp[i], s.ns, s.nxy, o, k) : slp_uniform(P, s.nxy, o, k);
  }
  if (!ok) k = 0;
  const float nan = slp_nan();
  for (int j = k; j < S; ++j) o.put(j, nan, nan, nan);
  nst[i] = k;
  if (statusp) statusp[i] = ok ? CRB_SLP_OK : CRB_SLP_OUT_OF_RANGE;
}

// The table is read straight from global memory: every thread of a warp reads the same row at the same time, so
// each load is one broadcast from L1, and no row cap is needed.
__global__ void __launch_bounds__(SLP_BLOCK)
crb_slp_search_kernel(int64_t n, const float* __restrict__ tgt, const float* __restrict__ table, int rows,
                      const float* __restrict__ k0, float* __restrict__ param, int32_t* __restrict__ rowp) {
  const int64_t i = (int64_t)blockIdx.x * SLP_BLOCK + threadIdx.x;
  if (i >= n) return;
  const float tx = tgt[i], ty = tgt[n + i], tyaw = tgt[2 * n + i];
  float best = FLT_MAX;
  int br = -1;
#pragma unroll 4
  for (int r = 0; r < rows; ++r) {
    const float* row = table + 6 * (int64_t)r;
    const float dx = __fsub_rn(tx, __ldg(row)), dy = __fsub_rn(ty, __ldg(row + 1)),
                dyaw = __fsub_rn(tyaw, __ldg(row + 2));
    // std::sqrt(dx * dx + dy * dy + dyaw * dyaw) on floats; compared as the rounded root, as the reference does
    const float d = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dyaw, dyaw)));
    if (d < best) {
      best = d;
      br = r;
    }
  }
  const float nan = slp_nan();
  const bool hit = br >= 0;
  param[i] = hit ? __fsqrt_rn(__fadd_rn(__fmul_rn(tx, tx), __fmul_rn(ty, ty))) : nan;
  param[n + i] = hit ? (k0 ? k0[i] : 0.0f) : nan;
  param[2 * n + i] = hit ? table[6 * (int64_t)br + 4] : nan;
  param[3 * n + i] = hit ? table[6 * (int64_t)br + 5] : nan;
  if (rowp) rowp[i] = br;
}

// S of crb.h, or -1 after setting the error string
static int slp_states(const crb_slp_sampler* s) {
  if (s == nullptr) {
    crb_set_error("crb_slp: invalid argument: sampler is NULL");
    return -1;
  }
  const bool polar = s->kind == CRB_SLP_UNIFORM || s->kind == CRB_SLP_BIASED;
  const char* bad = nullptr;
  if (!polar && s->kind != CRB_SLP_LANE) bad = "kind must be CRB_SLP_UNIFORM, CRB_SLP_BIASED or CRB_SLP_LANE";
  else if (s->nxy < 1 || s->nxy > CRB_SLP_MAX_NXY) bad = "nxy must be in [1, CRB_SLP_MAX_NXY]";
  else if (polar && (s->nh < 1 || s->nh > CRB_SLP_MAX_NH)) bad = "nh must be in [1, CRB_SLP_MAX_NH]";
  else if (s->kind == CRB_SLP_BIASED && (s->ns < 0 || s->ns > CRB_SLP_MAX_NS)) bad = "ns must be in [0, CRB_SLP_MAX_NS]";
  if (bad) {
    crb_set_error("crb_slp: invalid argument: %s", bad);
    return -1;
  }
  const int64_t S = s->kind == CRB_SLP_UNIFORM  ? (int64_t)s->nxy * s->nh
                    : s->kind == CRB_SLP_BIASED ? (int64_t)(s->nxy - 1) * s->nh
                                                : (int64_t)s->nxy;
  if (S > CRB_SLP_MAX_STATES) {
    crb_set_error("crb_slp: invalid argument: states per query exceed CRB_SLP_MAX_STATES");
    return -1;
  }
  return (int)S;
}

extern "C" {

void crb_slp_default_params(crb_mptg_params* p, float* v) {
  // src/state_lattice_planner.cpp:22-24 (L, DS, CONST_V), :146-148 (cost_th_, h_step_, max_iter)
  if (p) {
    p->base_l = (float)1.0;
    p->ds = (float)0.1;
    p->max_iter = 100;
    p->cost_th = (float)0.1;
    p->h_step[0] = (float)0.5;
    p->h_step[1] = (float)0.02;
    p->h_step[2] = (float)0.02;
  }
  if (v) *v = (float)3.0;
}

int crb_slp_states_per_query(const crb_slp_sampler* s) { return slp_states(s); }

int crb_slp_sample_states_batched(crb_ctx* ctx, int64_t n_q, const crb_slp_sampler* s, const float* qp,
                                  float* target, int32_t* n_states, int32_t* status) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(n_q >= 0 && (n_q + SLP_BLOCK - 1) / SLP_BLOCK <= 0x7fffffff, "n_q out of range");
  const int S = slp_states(s);
  if (S < 0) return CRB_ERR_INVALID_ARG;
  CRB_REQUIRE(n_q <= INT64_MAX / (S > 0 ? S : 1) / 3, "n_q * S out of range");
  CRB_REQUIRE(n_q == 0 || (qp && n_states && (target || S == 0)), "qp, target or n_states is NULL");
  const int rc = crb_require_device(__func__);
  if (rc != CRB_OK) return rc;
  if (n_q == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  crb_slp_sample_kernel<<<crb_grid_for(n_q, SLP_BLOCK), SLP_BLOCK, 0, ctx->stream>>>(n_q, *s, S, qp, target,
                                                                                     n_states, status);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

int crb_slp_search_nearest_batched(crb_ctx* ctx, int64_t n, const float* target, const float* table, int rows,
                                   const float* k0, float* param, int32_t* row) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(n >= 0 && (n + SLP_BLOCK - 1) / SLP_BLOCK <= 0x7fffffff, "n out of range");
  CRB_REQUIRE(rows >= 1, "rows must be >= 1");
  CRB_REQUIRE(n == 0 || (target && table && param), "target, table or param is NULL");
  const int rc = crb_require_device(__func__);
  if (rc != CRB_OK) return rc;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  crb_slp_search_kernel<<<crb_grid_for(n, SLP_BLOCK), SLP_BLOCK, 0, ctx->stream>>>(n, target, table, rows, k0,
                                                                                   param, row);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

}  // extern "C"
