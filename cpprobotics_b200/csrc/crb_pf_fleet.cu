// crb_pf_fleet.cu — one complete particle-filter iteration for a fleet of independent filters in ONE launch
// (crb_pf_step_many_batched) for sm_90a.
//
// Replaces pf_localization() + resampling(), src/particle_filter.cpp:73-148, called once per robot with the robot's
// own control u and observation list z (:257-271).  Each robot's filter is np particles, columns [r*np, (r+1)*np) of
// the field-major arrays.
//
// Launch form: one warp per robot, FLEET_WARPS robots per CTA.  A warp stages its robot's observation rows, its
// predicted particles, its weights and its cumulative weights in its own slice of dynamic shared memory
// (pf_fleet_slice_bytes), then runs predict + weight (the two-lane routine of crb_pf_common.cuh, particles 2l and
// 2l + 1 of each 64-particle round in lane l), the weight sum, normalisation, the estimate moments around the robot's
// heaviest particle, Neff, the resampling decision, the cumulative weights and the gather, with warp shuffles and
// __syncwarp only: no global scan, no second launch.  The reductions have a fixed order (lane-sequential, then a
// fixed shuffle tree), so a robot's outputs do not depend on the launch shape or on the other robots.
#include "crb_pf_common.cuh"

#define FLEET_WARPS 8
#define FLEET_SMEM_MAX (227 * 1024)   // sm_90's opt-in dynamic shared memory per CTA

// per-warp slice: double d[64] (the result column, the pivot, the moments) | float lm[3 * CRB_PF_MAX_LANDMARKS] |
// float x[4][np] | float w[np] | float c[np]
#define FLEET_HEAD_FLOATS 320
static inline size_t pf_fleet_slice_bytes(int np) { return (FLEET_HEAD_FLOATS + (size_t)6 * np) * sizeof(float); }
static_assert((FLEET_HEAD_FLOATS + 6 * CRB_PF_FLEET_MAX_NP) * 4 <= FLEET_SMEM_MAX, "one robot's slice must fit a CTA");

struct PfFleetArgs {
  PfArgs a;                                   // the batch's constants, built by pf_fill_args as for crb_pf_step
  float nlp[CRB_PF_MAX_LANDMARKS + 1][2];     // a.nlp_hi / a.nlp_lo for a list of k rows (pf_fill_args' expression)
  int64_t n_robots, n_rows;
  int32_t np, n_sets;
  double inv_np;                              // 1.0 / (double)np
  uint32_t rs_lo, rs_hi;                      // resample_seed
  float nth;
  int slice_floats;                           // pf_fleet_slice_bytes(np) / 4
};

__global__ void __launch_bounds__(FLEET_WARPS * 32)
crb_pf_fleet_kernel(float* __restrict__ px, float* __restrict__ pw, float* __restrict__ px_next,
                    const float* __restrict__ u, const float* __restrict__ noise, const float* __restrict__ z,
                    const int64_t* __restrict__ z_off, const int32_t* __restrict__ z_of,
                    const float* __restrict__ uniforms, double* __restrict__ result, int32_t* __restrict__ status,
                    const __grid_constant__ PfFleetArgs fa) {
  extern __shared__ double s_dyn[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + wid;
  if (r >= fa.n_robots) return;
  const int np = fa.np;
  const int64_t nr = fa.n_robots;
  const int64_t N = nr * np;                 // leading dimension of the field-major arrays
  const int64_t base = r * np;
  float* slice = reinterpret_cast<float*>(s_dyn) + (size_t)wid * fa.slice_floats;
  double* s_d = reinterpret_cast<double*>(slice);   // [0..23] the result column, [24..27] the pivot, [32..46] moments
  float* s_lm = slice + 128;
  float* s_x = slice + FLEET_HEAD_FLOATS;
  float* s_w = s_x + 4 * np;
  float* s_c = s_w + np;

  int64_t zb, ze;
  if (!crb_obstacle_list(r, z_off, fa.n_sets, z_of, fa.n_rows, CRB_PF_MAX_LANDMARKS, zb, ze)) {
    if (lane < CRB_PF_RESULT_LEN) result[(int64_t)lane * nr + r] = __longlong_as_double(0x7ff8000000000000ll);
    if (status && lane == 0) status[r] = CRB_PF_FLEET_BAD_OBSERVATIONS;
    return;   // px, pw and px_next keep their values
  }
  const int n_lm = (int)(ze - zb);
  for (int i = lane; i < 3 * n_lm; i += 32) s_lm[i] = z[3 * zb + i];

  // the robot's constants: the batch's, with its own control and its own observation count (what pf_fill_args
  // gives crb_pf_step for prm->u = u_r and n_lm rows)
  PfArgs a = fa.a;
  a.u[0] = u[r];
  a.u[1] = u[nr + r];
  a.u_d[0] = (double)a.u[0];
  a.u_d[1] = (double)a.u[1];
  a.n_lm = n_lm;
  a.nlp_hi = fa.nlp[n_lm][0];
  a.nlp_lo = fa.nlp[n_lm][1];
  __syncwarp();

  // ---- predict + weight (:81-102): particles j and j + 1 in the two lanes; a lone last particle in both ----
  // The lane also keeps the heaviest of its raw weights (ties to the lower index; a NaN never wins), the pivot of the
  // moments below: per round the larger of its pair, and the pair's first particle.
  const float2 one = f2(a.one);
  double sw_d = 0.0;
  float bw = -INFINITY;
  int bp = 0;
  for (int p0 = 0; p0 < np; p0 += 64) {
    const int j = p0 + 2 * lane;
    if (j < np) {
      const bool two = j + 1 < np;
      const int k = two ? j + 1 : j;
      const int64_t gj = base + j, gk = base + k;
      float2 X0 = f2(px[gj], px[gk]), X1 = f2(px[N + gj], px[N + gk]);
      float2 X2 = f2(px[2 * N + gj], px[2 * N + gk]), X3 = f2(px[3 * N + gj], px[3 * N + gk]);
      const float2 W = f2(pw[gj], pw[gk]);
      float2 G0, G1;
      if (a.has_noise) {
        G0 = f2(noise[gj], noise[gk]);
        G1 = f2(noise[N + gj], noise[N + gk]);
      } else {
        philox_normal2(a.seed_lo, a.seed_hi, (uint64_t)gj, G0.x, G1.x);
        if (two) philox_normal2(a.seed_lo, a.seed_hi, (uint64_t)gk, G0.y, G1.y);
        else { G0.y = G0.x; G1.y = G1.x; }
      }
      pf_motion2(X0, X1, X2, X3, G0, G1, a, one);
      const float2 Wn = pf_weight2_rows(X0, X1, W, a, one, s_lm);
      s_x[j] = X0.x; s_x[np + j] = X1.x; s_x[2 * np + j] = X2.x; s_x[3 * np + j] = X3.x;
      s_w[j] = Wn.x;
      sw_d += (double)Wn.x;
      const float w2 = fmaxf(Wn.x, Wn.y);   // Wn.y is particle j again when it is the lone last one
      if (w2 > bw) { bw = w2; bp = j; }
      if (two) {
        s_x[k] = X0.y; s_x[np + k] = X1.y; s_x[2 * np + k] = X2.y; s_x[3 * np + k] = X3.y;
        s_w[k] = Wn.y;
        sw_d += (double)Wn.y;
      }
    }
  }
  // the heaviest particle of the lane: the first of its pair unless that one is lighter (or NaN)
  int bi = bw > -INFINITY && !(s_w[bp] == bw) ? bp + 1 : bp;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sw_d += __shfl_down_sync(0xffffffffu, sw_d, o);
    const float ow = __shfl_xor_sync(0xffffffffu, bw, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ow > bw || (ow == bw && oi < bi)) { bw = ow; bi = oi; }   // the same winner in every lane
  }
  sw_d = __shfl_sync(0xffffffffu, sw_d, 0);   // pw.sum() before the normalisation, the same bits in every lane
  __syncwarp();

  // ---- normalise (:104), cumulative weights (:111-118), sum of squares (:126), moments around the heaviest
  // particle: its normalised weight w_max >= 1/np and Var_f >= w_max (x_f - xEst_f)^2, so the pivot lies within
  // sqrt(np) standard deviations of the mean and the one-pass moments lose at most ~np 2^-52 of each variance to
  // cancellation, wherever the cloud and its outliers are.  All-zero or NaN weights keep particle 0 (NaN results). ----
  const float sw = (float)sw_d;              // pw.sum() is a float in the reference (:104)
  double piv[4];
#pragma unroll
  for (int f = 0; f < 4; ++f) piv[f] = (double)s_x[f * np + bi];
  double v[15], sq = 0.0, carry = 0.0;
#pragma unroll
  for (int q = 0; q < 15; ++q) v[q] = 0.0;
  for (int j0 = 0; j0 < np; j0 += 32) {
    const int j = j0 + lane;
    float wn = 0.0f;
    if (j < np) {
      wn = s_w[j] / sw;
      s_w[j] = wn;
    }
    const double wd = (double)wn;
    double incl = wd;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (j < np) {
      s_c[j] = (float)(carry + incl);
      sq += wd * wd;
      double x[4], wx[4];
#pragma unroll
      for (int f = 0; f < 4; ++f) {
        x[f] = (double)s_x[f * np + j] - piv[f];
        wx[f] = wd * x[f];
      }
      v[0] += wd;
#pragma unroll
      for (int f = 0; f < 4; ++f) v[1 + f] += wx[f];
      int q = 5;
#pragma unroll
      for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int rr = c; rr < 4; ++rr, ++q) v[q] = fma(wx[rr], x[c], v[q]);   // one rounding per term
    }
    carry += __shfl_sync(0xffffffffu, incl, 31);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sq += __shfl_down_sync(0xffffffffu, sq, o);
#pragma unroll
    for (int q = 0; q < 15; ++q) v[q] += __shfl_down_sync(0xffffffffu, v[q], o);
  }
  int doit = 0;
  if (lane == 0) {
#pragma unroll
    for (int f = 0; f < 4; ++f) s_d[24 + f] = piv[f];
#pragma unroll
    for (int q = 0; q < 15; ++q) s_d[32 + q] = v[q];
    pf_finalize_normalised(s_d + 32, s_d + 24, s_d);     // [0..19] xEst, PEst (:104-107)
    // float Neff = 1.0 / (pw^T pw) (:126): the 1x1 product is a float, the quotient a double narrowed
    const float neff = (float)(1.0 / (double)(float)sq);
    doit = neff < fa.nth ? 1 : 0;                        // :127
    s_d[20] = sw_d;
    s_d[21] = (double)neff;
    s_d[22] = doit ? 1.0 : 0.0;
    s_d[23] = sq;
  }
  doit = __shfl_sync(0xffffffffu, doit, 0);
  __syncwarp();
  if (lane < CRB_PF_RESULT_LEN) result[(int64_t)lane * nr + r] = s_d[lane];
  if (status && lane == 0) status[r] = CRB_PF_FLEET_OK;

  // ---- the predicted particles and the weights: normalised, or Ones()*1.0/NP after a resampling (:147) ----
  const float wu = (float)fa.inv_np;
  for (int j = lane; j < np; j += 32) {
#pragma unroll
    for (int f = 0; f < 4; ++f) px[f * N + base + j] = s_x[f * np + j];
    pw[base + j] = doit ? wu : s_w[j];
  }
  if (!doit) {   // Neff >= NTh: px_next is a copy
    for (int j = lane; j < np; j += 32) {
#pragma unroll
      for (int f = 0; f < 4; ++f) px_next[f * N + base + j] = s_x[f * np + j];
    }
    return;
  }
  // ---- resampling (:128-147): resampleid_j = j/NP + U_j/NP with the running maximum of crb_pf_step's gather
  // (resampleid_{j-1} and resampleid_j can be inverted by the rounding of j/NP); the first index whose cumulative
  // weight reaches it, capped at NP-1 (:136-143).  s_w holds the resampleids once the weights are written. ----
  __syncwarp();
  const double n_d = (double)np;
  for (int j = lane; j < np; j += 32) {
    const float U = uniforms ? uniforms[base + j] : philox_uniform12(fa.rs_lo, fa.rs_hi, (uint64_t)(base + j));
    s_w[j] = pf_resample_id_rcp(j, n_d, fa.inv_np, U);
  }
  __syncwarp();
  for (int j = lane; j < np; j += 32) {
    const float rid = j > 0 ? fmaxf(s_w[j], s_w[j - 1]) : s_w[0];
    int lo = 0, hi = np - 1;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (rid > s_c[mid]) lo = mid + 1; else hi = mid;
    }
#pragma unroll
    for (int f = 0; f < 4; ++f) px_next[f * N + base + j] = s_x[f * np + lo];
  }
}

extern "C" int crb_pf_step_many_batched(crb_ctx* ctx, int64_t n_robots, int32_t np, float* px, float* pw,
                                        float* px_next, const float* u, const float* noise, uint64_t seed,
                                        const float* z, int64_t n_rows, const int64_t* z_off, int32_t n_sets,
                                        const int32_t* z_of, const crb_pf_params* prm, const float* uniforms,
                                        uint64_t resample_seed, float nth, double* result, int32_t* status) {
  CRB_REQUIRE(ctx != nullptr && prm != nullptr, "ctx / prm is NULL");
  CRB_REQUIRE(np >= 1 && np <= CRB_PF_FLEET_MAX_NP, "np out of range");
  CRB_REQUIRE(n_robots >= 0 && n_robots <= ((int64_t)1 << 40) / np && n_robots <= 0x7fffffff, "n_robots out of range");
  CRB_REQUIRE(n_sets >= 1 && n_rows >= 0, "n_sets must be >= 1 and n_rows >= 0");
  CRB_REQUIRE(n_robots == 0 || (z_off && z_of && (z || n_rows == 0)), "z, z_off or z_of is NULL");
  CRB_REQUIRE(n_robots == 0 || (px && pw && px_next && u && result), "NULL array");
  CRB_REQUIRE(n_robots == 0 || px != px_next, "px and px_next must be different arrays");
  const int rc = crb_require_device(__func__);
  if (rc != CRB_OK) return rc;
  if (n_robots == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  PfFleetArgs fa;
  memset(&fa, 0, sizeof(fa));
  pf_fill_args(&fa.a, noise, seed, nullptr, 0, prm);
  for (int k = 0; k <= CRB_PF_MAX_LANDMARKS; ++k) {
    const double nlp = -(double)k * log(fa.a.pre);
    fa.nlp[k][0] = (float)nlp;
    fa.nlp[k][1] = (float)(nlp - (double)fa.nlp[k][0]);
  }
  fa.n_robots = n_robots;
  fa.n_rows = n_rows;
  fa.np = np;
  fa.n_sets = n_sets;
  fa.inv_np = 1.0 / (double)np;
  fa.rs_lo = (uint32_t)resample_seed;
  fa.rs_hi = (uint32_t)(resample_seed >> 32);
  fa.nth = nth;
  const size_t slice = pf_fleet_slice_bytes(np);
  fa.slice_floats = (int)(slice / sizeof(float));
  // FLEET_WARPS robots per CTA, or as many as the CTA's shared memory holds (np above 1157)
  const int wpc = (int)(FLEET_SMEM_MAX / slice) < FLEET_WARPS ? (int)(FLEET_SMEM_MAX / slice) : FLEET_WARPS;
  const size_t smem = slice * wpc;
  if (!ctx->pf_fleet_attr_set) {   // once per context, to the largest slice set any np needs: no per-call host cost,
                                   // and no call can lower the limit between another call's set and its launch
    CRB_CUDA(cudaFuncSetAttribute(crb_pf_fleet_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FLEET_SMEM_MAX));
    ctx->pf_fleet_attr_set = 1;
  }
  const int64_t blocks = (n_robots + wpc - 1) / wpc;
  crb_pf_fleet_kernel<<<(unsigned)blocks, wpc * 32, smem, ctx->stream>>>(
      px, pw, px_next, u, noise, z, z_off, z_of, uniforms, result, status, fa);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}
