// crb_mpc.cu — batched bicycle-model MPC solve for sm_90a.
//
// Replaces mpc_solve() + FG_EVAL of the reference, src/model_predictive_control.cpp:188-346 (the
// CppAD + IPOPT solve of the speed-and-steering NLP), for n independent agents per launch, plus the
// plant step update() :69-81 and the reference-trajectory lookup calc_ref_trajectory() :130-170 /
// calc_nearest_index() :107-127.
//
// Algorithm (BASELINE.json north_star: "horizon-T linearised dynamics, QP cost, Riccati factorise-
// and-solve replacing IPOPT"): box-constrained DDP on the reference NLP.  Each outer iteration
// linearises the dynamics :242-245 along the current roll-out (with their exact second derivatives),
// runs a Riccati recursion on the (state, previous input) augmented system so that the input-rate
// cost :207-210 is handled exactly, takes a projected-Newton step of the 2-D box QP of every stage in
// closed form (|delta|, |a| and the speed limits :288-301 folded into a bound on a_t; the stage
// Hessian may be indefinite), and rolls the clamped non-linear dynamics forward with step halving until the cost decreases
// (one Gauss-Newton retry if the Newton direction gives no decrease).  The executable specification is
// oracle/crb_oracle_mpc.c; this kernel reproduces it BIT FOR BIT (explicit fmaf, -fmad=false,
// polynomial sin/cos, IEEE divide/sqrt), so status words and iteration counts match exactly.
//
// Mapping: ONE THREAD PER PROBLEM (workspace CTA-interleaved, see MPC_BLOCK below).  The matrices are 4x4 / 2x4 / 2x2 with five non-trivial entries
// in A and two in B: a warp per problem would idle >80 % of its lanes and pay shuffles for every
// product, whereas a thread per problem keeps the whole stage in registers, runs pure FFMA with
// ample ILP, and makes every global access a coalesced 128-byte line because all per-problem data
// (trajectories, gains) live in SoA scratch arrays indexed [item][problem].  At the BASELINE size
// (65 536 agents, 128 threads per CTA, <= 128 registers) the whole batch is resident in one wave.
#include <math.h>
#include <stdlib.h>

#include "crb_common.cuh"

#include "crb_mpc_core.cuh"
#include "crb_plant.cuh"
#include "crb_mpc_tasks.cuh"

// Thread-per-problem kernel (first generation; CRB_MPC_VARIANT=0): solver workspace in global memory,
// CTA-interleaved.  A CTA of MPC_BLOCK threads owns a contiguous slab [item][MPC_BLOCK]; thread t of the
// CTA reads item k at slab[k*MPC_BLOCK + t].  Accesses stay coalesced (MPC_BLOCK consecutive floats per
// item) and every per-thread offset is a COMPILE-TIME constant times the item index.
#define MPC_BLOCK 128
#define LS MPC_BLOCK

// ---- backward sweep -------------------------------------------------------------------------------
// X [4T][n], U [2(T-1)][n] (field 2t+c, c = 0 delta, 1 a), xref [4T][n] (course frame; ox, oy are
// subtracted on the fly), gains out G [14(T-1)][n].
// X [4T], U [2(T-1)] (item 2t+c, c = 0 delta, 1 a), XR [4T] (reference, already translated by
// (ox, oy)), gains out G [14(T-1)]: thread pointers into the CTA-interleaved workspace, item stride LS.
// L2 prefetch of one workspace word's 128-byte line (the warp's 32 lanes share it): no register, no wait.
__device__ __forceinline__ void pf_l2(const float* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

template <int PFD>
__device__ __forceinline__ void backward_sweep(int T, const float* __restrict__ X,
                                               const float* __restrict__ U,
                                               const float* __restrict__ XR, const MpcP& p,
                                               bool gn, float* __restrict__ G) {
  const int N = T - 1;
  const float R2[2] = {2.0f * p.w_delta, 2.0f * p.w_a};
  const float Rd2[2] = {2.0f * p.w_ddelta, 2.0f * p.w_da};
  const float Q2[4] = {2.0f * p.wq[0], 2.0f * p.wq[1], 2.0f * p.wq[2], 2.0f * p.wq[3]};
  const float dt = p.dt;
  float Pxx[4][4], Pxw[4][2], Pww[2][2], px[4], pw[2];
#pragma unroll
  for (int a = 0; a < 4; ++a) {
#pragma unroll
    for (int b = 0; b < 4; ++b) Pxx[a][b] = a == b ? Q2[a] : 0.0f;
    Pxw[a][0] = 0.0f; Pxw[a][1] = 0.0f;
  }
  Pww[0][0] = Pww[0][1] = Pww[1][0] = Pww[1][1] = 0.0f;
  pw[0] = pw[1] = 0.0f;
#pragma unroll
  for (int k = 0; k < 4; ++k) px[k] = Q2[k] * (X[(N * 4 + k) * LS] - XR[(N * 4 + k) * LS]);
  // Software pipeline: the operands of stage t-1 are requested at the top of stage t so that their
  // L2/HBM latency hides under stage t's arithmetic (the sweep is a 19-long dependent chain).
  float ut[2];                   // U[t]
  float xt[4], xr[4], um[2];     // X[t], xref[t] (translated), U[t-1]
  ut[0] = U[((N - 1) * 2 + 0) * LS];
  ut[1] = U[((N - 1) * 2 + 1) * LS];
  auto load_stage = [&](int t, float (&x_)[4], float (&r_)[4], float (&m_)[2]) {
    const float* xs = X + t * 4 * LS;
    const float* rs = XR + t * 4 * LS;
    const float* us = U + (t - 1) * 2 * LS;
#pragma unroll
    for (int k = 0; k < 4; ++k) x_[k] = xs[k * LS];
    if (t >= 1) {
#pragma unroll
      for (int k = 0; k < 4; ++k) r_[k] = rs[k * LS];
      m_[0] = us[0];
      m_[1] = us[LS];
    } else {
      r_[0] = r_[1] = r_[2] = r_[3] = 0.0f;
      m_[0] = m_[1] = 0.0f;
    }
  };
  load_stage(N - 1, xt, xr, um);

  for (int t = N - 1; t >= 0; --t) {
    const bool hr = t >= 1;
    float xt_n[4] = {0.0f, 0.0f, 0.0f, 0.0f}, xr_n[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    float um_n[2] = {0.0f, 0.0f};
    if (t >= 1) load_stage(t - 1, xt_n, xr_n, um_n);
    if (PFD > 0 && t - 1 - PFD >= 0) {   // stage t-1-PFD: pull its lines into L2 now
      const int tp = t - 1 - PFD;
#pragma unroll
      for (int k = 0; k < 4; ++k) { pf_l2(X + (tp * 4 + k) * LS); pf_l2(XR + (tp * 4 + k) * LS); }
      if (tp >= 1) { pf_l2(U + ((tp - 1) * 2 + 0) * LS); pf_l2(U + ((tp - 1) * 2 + 1) * LS); }
    }
    const float v = xt[3];
    float s, c, sd, cd;
    crb_sincosf(xt[2], s, c);
    crb_sincosf(ut[0], sd, cd);
    const float tn = sd / cd;
    const float kap = tn * p.inv_wb;
    const float vdt = v * dt;
    const float bv = (dt * p.inv_wb) * fmaf(tn, tn, 1.0f);
    const float B20 = v * bv;
    // A = I + {(0,2) a02, (0,3) a03, (1,2) a12, (1,3) a13, (2,3) a23};  B = {(2,0) B20, (3,1) dt}
    const float a02 = -(vdt * s), a03 = c * dt, a12 = vdt * c, a13 = s * dt, a23 = kap * dt;

    // gradients: qx = A^T px (+ Q2 (x - r)), qu = R2 u (+ Rd2 du) + B^T px + pw, qw = -Rd2 du
    float qx[4], qu[2], qw[2], du[2] = {0.0f, 0.0f};
    qx[0] = px[0];
    qx[1] = px[1];
    qx[2] = px[2] + fmaf(a12, px[1], a02 * px[0]);
    qx[3] = px[3] + fmaf(a23, px[2], fmaf(a13, px[1], a03 * px[0]));
    if (hr) {
#pragma unroll
      for (int k = 0; k < 4; ++k) qx[k] = fmaf(Q2[k], xt[k] - xr[k], qx[k]);
    }
    const float BtPx[2] = {B20 * px[2], dt * px[3]};
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      if (hr) du[a] = ut[a] - um[a];
      float g = R2[a] * ut[a];
      if (hr) g = fmaf(Rd2[a], du[a], g);
      g = g + BtPx[a];
      g = g + pw[a];
      qu[a] = g;
      qw[a] = hr ? -(Rd2[a] * du[a]) : 0.0f;
    }
    const float hyy = gn ? 0.0f : -(vdt * fmaf(px[1], s, px[0] * c));
    const float hyv = gn ? 0.0f : dt * fmaf(px[1], c, -(px[0] * s));

    // G = Pxx A (structural zeros/ones of A skipped; same term order as the dense product)
    float Gm[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      Gm[a][0] = Pxx[a][0];
      Gm[a][1] = Pxx[a][1];
      Gm[a][2] = Pxx[a][2] + fmaf(Pxx[a][1], a12, Pxx[a][0] * a02);
      Gm[a][3] = Pxx[a][3] + fmaf(Pxx[a][2], a23, fmaf(Pxx[a][1], a13, Pxx[a][0] * a03));
    }
    // Qxx = A^T G (+ Q2) (+ second-order terms), lower triangle only
    float Qxx[4][4];
    Qxx[0][0] = Gm[0][0];
    Qxx[1][0] = Gm[1][0];
    Qxx[1][1] = Gm[1][1];
#pragma unroll
    for (int b = 0; b < 3; ++b) Qxx[2][b] = Gm[2][b] + fmaf(a12, Gm[1][b], a02 * Gm[0][b]);
#pragma unroll
    for (int b = 0; b < 4; ++b)
      Qxx[3][b] = Gm[3][b] + fmaf(a23, Gm[2][b], fmaf(a13, Gm[1][b], a03 * Gm[0][b]));
    if (hr) {
#pragma unroll
      for (int a = 0; a < 4; ++a) Qxx[a][a] = Qxx[a][a] + Q2[a];
    }
    Qxx[2][2] = Qxx[2][2] + hyy;
    Qxx[3][2] = Qxx[3][2] + hyv;
    // Qux = B^T G + Pwx A (+ second-order)
    float Qux[2][4];
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const float w0 = Pxw[0][a], w1 = Pxw[1][a], w2 = Pxw[2][a], w3 = Pxw[3][a];
      const float W0 = w0, W1 = w1;
      const float W2 = w2 + fmaf(w1, a12, w0 * a02);
      const float W3 = w3 + fmaf(w2, a23, fmaf(w1, a13, w0 * a03));
      const float bb = a == 0 ? B20 : dt;
      const int row = a == 0 ? 2 : 3;
      Qux[a][0] = bb * Gm[row][0] + W0;
      Qux[a][1] = bb * Gm[row][1] + W1;
      Qux[a][2] = bb * Gm[row][2] + W2;
      Qux[a][3] = bb * Gm[row][3] + W3;
    }
    if (!gn) Qux[0][3] = fmaf(px[2], bv, Qux[0][3]);
    // Quu = Luu + B^T Pxx B + B^T Pxw + Pwx B + Pww (+ second-order)
    const float PB20 = Pxx[2][2] * B20, PB21 = Pxx[2][3] * dt, PB31 = Pxx[3][3] * dt;
    const float BtPB00 = B20 * PB20, BtPB01 = B20 * PB21, BtPB11 = dt * PB31;
    const float BtPxw00 = B20 * Pxw[2][0], BtPxw01 = B20 * Pxw[2][1];
    const float BtPxw10 = dt * Pxw[3][0], BtPxw11 = dt * Pxw[3][1];
    const float L0 = hr ? R2[0] + Rd2[0] : R2[0];
    const float L1 = hr ? R2[1] + Rd2[1] : R2[1];
    float Q00 = (((L0 + BtPB00) + BtPxw00) + BtPxw00) + Pww[0][0];
    const float Q01 = (((0.0f + BtPB01) + BtPxw01) + BtPxw10) + Pww[0][1];
    const float Q11 = (((L1 + BtPB11) + BtPxw11) + BtPxw11) + Pww[1][1];
    if (!gn) Q00 = fmaf(px[2], (2.0f * tn) * B20, Q00);
    const float Quw[2] = {hr ? -Rd2[0] : 0.0f, hr ? -Rd2[1] : 0.0f};
    const float Qww[2] = {hr ? Rd2[0] : 0.0f, hr ? Rd2[1] : 0.0f};

    float alo, ahi;
    bool lo_sp, hi_sp;
    a_bounds(v, p, alo, ahi, lo_sp, hi_sp);
    const float lo0 = -p.max_steer - ut[0], lo1 = alo - ut[1];
    const float hi0 = p.max_steer - ut[0], hi1 = ahi - ut[1];
    // Quu may be indefinite: projected-Newton box QP; gains from the regularised free-input Hessian,
    // value update (below) with the true Quu
    QpResult qp;
    box_qp2(Q00, Q01, Q11, qu[0], qu[1], lo0, lo1, hi0, hi1, qp);
    const float k0 = qp.k0, k1 = qp.k1;
    const bool cl0 = qp.cl0, cl1 = qp.cl1;
    const float H00 = qp.H00, H11 = qp.H11, H01 = Q01;
    const float idet = qp.idet, ih00 = qp.ih00, ih11 = qp.ih11;
    float Kx[2][4], Kw[2][2];
#pragma unroll
    for (int b = 0; b < 4; ++b) { Kx[0][b] = 0.0f; Kx[1][b] = 0.0f; }
    Kw[0][0] = Kw[0][1] = Kw[1][0] = Kw[1][1] = 0.0f;
    if (cl1) {
      const bool at_lo = k1 <= lo1;
      if ((at_lo && lo_sp) || (!at_lo && hi_sp)) Kx[1][3] = -p.inv_dt;
    }
    if (!cl0 && !cl1) {
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        Kx[0][b] = fmaf(H01, Qux[1][b], -(H11 * Qux[0][b])) * idet;
        Kx[1][b] = fmaf(H01, Qux[0][b], -(H00 * Qux[1][b])) * idet;
      }
      Kw[0][0] = fmaf(H01, 0.0f, -(H11 * Quw[0])) * idet;
      Kw[1][0] = fmaf(H01, Quw[0], -(H00 * 0.0f)) * idet;
      Kw[0][1] = fmaf(H01, Quw[1], -(H11 * 0.0f)) * idet;
      Kw[1][1] = fmaf(H01, 0.0f, -(H00 * Quw[1])) * idet;
    } else if (!cl0) {  // delta free (j = 0), a clamped (i = 1)
#pragma unroll
      for (int b = 0; b < 4; ++b) Kx[0][b] = -(fmaf(H01, Kx[1][b], Qux[0][b]) * ih00);
      Kw[0][0] = -(fmaf(H01, Kw[1][0], Quw[0]) * ih00);
      Kw[0][1] = -(fmaf(H01, Kw[1][1], 0.0f) * ih00);
    } else if (!cl1) {  // a free (j = 1), delta clamped (i = 0)
#pragma unroll
      for (int b = 0; b < 4; ++b) Kx[1][b] = -(fmaf(H01, Kx[0][b], Qux[1][b]) * ih11);
      Kw[1][0] = -(fmaf(H01, Kw[0][0], 0.0f) * ih11);
      Kw[1][1] = -(fmaf(H01, Kw[0][1], Quw[1]) * ih11);
    }
    // store gains for the forward sweeps
    {
      float* g = G + t * NGAIN * LS;
      g[0 * LS] = k0; g[1 * LS] = k1;
#pragma unroll
      for (int b = 0; b < 4; ++b) { g[(2 + b) * LS] = Kx[0][b]; g[(6 + b) * LS] = Kx[1][b]; }
      g[10 * LS] = Kw[0][0]; g[11 * LS] = Kw[0][1]; g[12 * LS] = Kw[1][0]; g[13 * LS] = Kw[1][1];
    }
    // value-function update for du = k + Kx dx + Kw dw with the TRUE Quu
    const float m0 = fmaf(Q01, k1, fmaf(Q00, k0, qu[0]));
    const float m1 = fmaf(Q11, k1, fmaf(Q01, k0, qu[1]));
    float Mx[2][4], Mw[2][2];
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      Mx[0][b] = fmaf(Q01, Kx[1][b], fmaf(Q00, Kx[0][b], Qux[0][b]));
      Mx[1][b] = fmaf(Q11, Kx[1][b], fmaf(Q01, Kx[0][b], Qux[1][b]));
    }
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      Mw[0][b] = fmaf(Q01, Kw[1][b], fmaf(Q00, Kw[0][b], b == 0 ? Quw[0] : 0.0f));
      Mw[1][b] = fmaf(Q11, Kw[1][b], fmaf(Q01, Kw[0][b], b == 1 ? Quw[1] : 0.0f));
    }
    float npx[4], npw[2];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      float acc = qx[a];
      acc = fmaf(Kx[0][a], m0, acc);
      acc = fmaf(Kx[1][a], m1, acc);
      acc = fmaf(Qux[0][a], k0, acc);
      acc = fmaf(Qux[1][a], k1, acc);
      npx[a] = acc;
    }
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      float acc = qw[b];
      acc = fmaf(Kw[0][b], m0, acc);
      acc = fmaf(Kw[1][b], m1, acc);
      acc = fmaf(Quw[b], b == 0 ? k0 : k1, acc);
      npw[b] = acc;
    }
    float nPxx[4][4], nPxw[4][2], nPww[2][2];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
#pragma unroll
      for (int b = 0; b <= a; ++b) {
        float acc = Qxx[a][b];
        acc = fmaf(Kx[0][a], Mx[0][b], acc);
        acc = fmaf(Kx[1][a], Mx[1][b], acc);
        acc = fmaf(Qux[0][a], Kx[0][b], acc);
        acc = fmaf(Qux[1][a], Kx[1][b], acc);
        nPxx[a][b] = acc;
        nPxx[b][a] = acc;
      }
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        float acc = Kx[0][a] * Mw[0][b];
        acc = fmaf(Kx[1][a], Mw[1][b], acc);
        acc = fmaf(Qux[0][a], Kw[0][b], acc);
        acc = fmaf(Qux[1][a], Kw[1][b], acc);
        nPxw[a][b] = acc;
      }
    }
#pragma unroll
    for (int a = 0; a < 2; ++a) {
#pragma unroll
      for (int b = 0; b <= a; ++b) {
        float acc = a == b ? Qww[a] : 0.0f;
        acc = fmaf(Kw[0][a], Mw[0][b], acc);
        acc = fmaf(Kw[1][a], Mw[1][b], acc);
        acc = fmaf(Quw[a], Kw[a][b], acc);
        nPww[a][b] = acc;
        nPww[b][a] = acc;
      }
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
#pragma unroll
      for (int b = 0; b < 4; ++b) Pxx[a][b] = nPxx[a][b];
      Pxw[a][0] = nPxw[a][0]; Pxw[a][1] = nPxw[a][1];
      px[a] = npx[a];
    }
    Pww[0][0] = nPww[0][0]; Pww[0][1] = nPww[0][1]; Pww[1][0] = nPww[1][0]; Pww[1][1] = nPww[1][1];
    pw[0] = npw[0]; pw[1] = npw[1];
    ut[0] = um[0]; ut[1] = um[1];
#pragma unroll
    for (int k = 0; k < 4; ++k) { xt[k] = xt_n[k]; xr[k] = xr_n[k]; }
    um[0] = um_n[0]; um[1] = um_n[1];
  }
}

// ---- forward sweep: clamped roll-out under the affine policy; returns dJ and sum|du| ----------------
template <int PFD>
__device__ __forceinline__ void forward_sweep(int T, float yaw0, float v0,
                                              const float* __restrict__ X,
                                              const float* __restrict__ U,
                                              const float* __restrict__ XR,
                                              const float* __restrict__ G, float alpha,
                                              const MpcP& p, float* __restrict__ Xn,
                                              float* __restrict__ Un, float& dJ_out,
                                              float& du_out) {
  float dJ = 0.0f, dus = 0.0f;
  float xn[4] = {0.0f, 0.0f, yaw0, v0};   // Xn[t]
  float xo[4] = {0.0f, 0.0f, yaw0, v0};   // X[t]  (both roll-outs start at x0)
  float unm[2] = {0.0f, 0.0f}, uom[2] = {0.0f, 0.0f};  // Un[t-1], U[t-1]
#pragma unroll
  for (int k = 0; k < 4; ++k) Xn[k * LS] = xn[k];
  const float wu[2] = {p.w_delta, p.w_a};
  const float wd[2] = {p.w_ddelta, p.w_da};
  float uo[2], gk[NGAIN], xo1[4], xr1[4];
  auto load_stage = [&](int t, float (&uo_)[2], float (&gk_)[NGAIN], float (&xo1_)[4],
                        float (&xr1_)[4]) {
    const float* g = G + t * NGAIN * LS;
    const float* us = U + t * 2 * LS;
    const float* xs = X + (t + 1) * 4 * LS;
    const float* rs = XR + (t + 1) * 4 * LS;
    uo_[0] = us[0];
    uo_[1] = us[LS];
#pragma unroll
    for (int j = 0; j < NGAIN; ++j) gk_[j] = g[j * LS];
#pragma unroll
    for (int k = 0; k < 4; ++k) { xo1_[k] = xs[k * LS]; xr1_[k] = rs[k * LS]; }
  };
  load_stage(0, uo, gk, xo1, xr1);
  for (int t = 0; t < T - 1; ++t) {
    // software pipeline: request stage t+1's operands before stage t's arithmetic
    float uo_n[2] = {0.0f, 0.0f}, gk_n[NGAIN], xo1_n[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    float xr1_n[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
    for (int j = 0; j < NGAIN; ++j) gk_n[j] = 0.0f;
    if (t + 1 < T - 1) load_stage(t + 1, uo_n, gk_n, xo1_n, xr1_n);
    if (PFD > 0 && t + 1 + PFD < T - 1) {   // stage t+1+PFD: pull its lines into L2 now
      const int tp = t + 1 + PFD;
      pf_l2(U + (tp * 2 + 0) * LS);
      pf_l2(U + (tp * 2 + 1) * LS);
#pragma unroll
      for (int j = 0; j < NGAIN; ++j) pf_l2(G + (tp * NGAIN + j) * LS);
#pragma unroll
      for (int k = 0; k < 4; ++k) { pf_l2(X + ((tp + 1) * 4 + k) * LS); pf_l2(XR + ((tp + 1) * 4 + k) * LS); }
    }
    float dx[4], dw[2] = {0.0f, 0.0f};
#pragma unroll
    for (int k = 0; k < 4; ++k) dx[k] = xn[k] - xo[k];
    if (t >= 1) { dw[0] = unm[0] - uom[0]; dw[1] = unm[1] - uom[1]; }
    float u[2];
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      float acc = fmaf(alpha, gk[a], uo[a]);
#pragma unroll
      for (int b = 0; b < 4; ++b) acc = fmaf(gk[2 + 4 * a + b], dx[b], acc);
#pragma unroll
      for (int b = 0; b < 2; ++b) acc = fmaf(gk[10 + 2 * a + b], dw[b], acc);
      u[a] = acc;
    }
    u[0] = clampf(u[0], -p.max_steer, p.max_steer);
    float alo, ahi;
    bool s0, s1;
    a_bounds(xn[3], p, alo, ahi, s0, s1);
    u[1] = clampf(u[1], alo, ahi);
    Un[(t * 2 + 0) * LS] = u[0];
    Un[(t * 2 + 1) * LS] = u[1];
    float xn1[4];
    dyn_step(xn, u[0], u[1], p, xn1);
#pragma unroll
    for (int k = 0; k < 4; ++k) Xn[((t + 1) * 4 + k) * LS] = xn1[k];
    // cost difference, term by term: w (q' - q)(q' + q)
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const float d = u[a] - uo[a], sm = u[a] + uo[a];
      dJ = fmaf(wu[a] * d, sm, dJ);
      dus = dus + fabsf(d);
    }
    if (t >= 1) {
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        const float qn = u[a] - unm[a], qo = uo[a] - uom[a];
        dJ = fmaf(wd[a] * (qn - qo), qn + qo, dJ);
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float en = xn1[k] - xr1[k], eo = xo1[k] - xr1[k];
      dJ = fmaf(p.wq[k] * (xn1[k] - xo1[k]), en + eo, dJ);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) { xn[k] = xn1[k]; xo[k] = xo1[k]; }
    unm[0] = u[0]; unm[1] = u[1]; uom[0] = uo[0]; uom[1] = uo[1];
    uo[0] = uo_n[0]; uo[1] = uo_n[1];
#pragma unroll
    for (int j = 0; j < NGAIN; ++j) gk[j] = gk_n[j];
#pragma unroll
    for (int k = 0; k < 4; ++k) { xo1[k] = xo1_n[k]; xr1[k] = xr1_n[k]; }
  }
  dJ_out = dJ;
  du_out = dus;
}

// fg[0] (:199-250) on a stored roll-out, same term order as direct_cost() in the oracle
__device__ __forceinline__ float direct_cost(int T, const float* __restrict__ X,
                                             const float* __restrict__ U,
                                             const float* __restrict__ XR, const MpcP& p) {
  float J = 0.0f;
  float um[2] = {0.0f, 0.0f};
  for (int t = 0; t < T - 1; ++t) {
    const float d = U[(t * 2 + 0) * LS], a = U[(t * 2 + 1) * LS];
    J = fmaf(p.w_delta * d, d, J);
    J = fmaf(p.w_a * a, a, J);
    if (t >= 1) {
      const float dd = d - um[0], da = a - um[1];
      J = fmaf(p.w_ddelta * dd, dd, J);
      J = fmaf(p.w_da * da, da, J);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float e = X[((t + 1) * 4 + k) * LS] - XR[((t + 1) * 4 + k) * LS];
      J = fmaf(p.wq[k] * e, e, J);
    }
    um[0] = d; um[1] = a;
  }
  return J;
}

// Workspace items per problem: XA [4T] XB [4T] UA [2N] UB [2N] G [14N] XR [4T]
__host__ __device__ inline int mpc_ws_items(int T) { return 12 * T + (4 + NGAIN) * (T - 1); }

template <int PFD>
__global__ void __launch_bounds__(MPC_BLOCK, 4)
crb_mpc_solve_kernel(int64_t count, int64_t ld_in, int T, const float* __restrict__ x0,
                     const float* __restrict__ xref, const float* __restrict__ u_init,
                     float* __restrict__ ws, int64_t ld_out, float* __restrict__ sol,
                     float* __restrict__ u0, float* __restrict__ cost, int32_t* __restrict__ status,
                     int32_t* __restrict__ iters, const MpcP p) {
  const int64_t i = (int64_t)blockIdx.x * MPC_BLOCK + threadIdx.x;
  if (i >= count) return;
  const int64_t n = ld_in;
  const int N = T - 1;
  // this thread's column of the CTA's workspace slab
  float* S = ws + (size_t)blockIdx.x * mpc_ws_items(T) * MPC_BLOCK + threadIdx.x;
  float* X = S;
  float* Xn = X + 4 * T * LS;
  float* U = Xn + 4 * T * LS;
  float* Un = U + 2 * N * LS;
  float* G = Un + 2 * N * LS;
  float* XR = G + NGAIN * N * LS;
  const float ox = x0[0 * n + i], oy = x0[1 * n + i];
  const float yaw0 = x0[2 * n + i], v0 = x0[3 * n + i];
  // reference trajectory into the workspace, translated to the frame of the initial position
  for (int t = 0; t < T; ++t) {
    XR[(t * 4 + 0) * LS] = xref[((int64_t)t * 4 + 0) * n + i] - ox;
    XR[(t * 4 + 1) * LS] = xref[((int64_t)t * 4 + 1) * n + i] - oy;
    XR[(t * 4 + 2) * LS] = xref[((int64_t)t * 4 + 2) * n + i];
    XR[(t * 4 + 3) * LS] = xref[((int64_t)t * 4 + 3) * n + i];
  }
  // initial clamped roll-out (cold start: zeros, :266-269)
  {
    float x[4] = {0.0f, 0.0f, yaw0, v0};
#pragma unroll
    for (int k = 0; k < 4; ++k) X[k * LS] = x[k];
    for (int t = 0; t < N; ++t) {
      float d = u_init ? u_init[(int64_t)t * n + i] : 0.0f;
      float a = u_init ? u_init[(int64_t)(N + t) * n + i] : 0.0f;
      d = clampf(d, -p.max_steer, p.max_steer);
      float alo, ahi;
      bool s0, s1;
      a_bounds(x[3], p, alo, ahi, s0, s1);
      a = clampf(a, alo, ahi);
      U[(t * 2 + 0) * LS] = d;
      U[(t * 2 + 1) * LS] = a;
      float x1[4];
      dyn_step(x, d, a, p, x1);
#pragma unroll
      for (int k = 0; k < 4; ++k) { x[k] = x1[k]; X[((t + 1) * 4 + k) * LS] = x1[k]; }
    }
  }
  int st = CRB_MPC_MAX_ITER, it_count = 0;
  const float J0 = direct_cost(T, X, U, XR, p);
  if (!(fabsf(J0) <= 3.0e38f)) {
    st = CRB_MPC_NONFINITE;
  } else {
    bool gn = false;  // Newton sweep; Gauss-Newton retry after a failed line search
    float Jc = J0;    // running cost
    while (it_count < p.max_iter) {
      backward_sweep<PFD>(T, X, U, XR, p, gn, G);
      ++it_count;
      bool accepted = false, tiny = false;
      int jacc = 0;
      float dJ = 0.0f, du = 0.0f, alpha = 1.0f;
      for (int j = 0; j <= p.max_ls; ++j) {
        forward_sweep<PFD>(T, yaw0, v0, X, U, XR, G, alpha, p, Xn, Un, dJ, du);
        if (j == 0) tiny = (du <= p.du_th) || (fabsf(dJ) <= p.j_tol * fabsf(Jc));
        if (dJ < 0.0f) { accepted = true; jacc = j; break; }
        if (tiny) break;
        alpha = alpha * 0.5f;
      }
      if (!accepted) {
        if (tiny) { st = CRB_MPC_CONVERGED; break; }
        if (!gn) { gn = true; continue; }
        st = CRB_MPC_NO_DESCENT;
        break;
      }
      gn = false;
      float* tx = X; X = Xn; Xn = tx;
      float* tu = U; U = Un; Un = tu;
      Jc = Jc + dJ;
      if ((jacc == 0 && tiny) || du <= p.du_th) { st = CRB_MPC_CONVERGED; break; }
    }
  }
  const float J = direct_cost(T, X, U, XR, p);
  if (!(fabsf(J) <= 3.0e38f)) st = CRB_MPC_NONFINITE;
  const int64_t m = ld_out;
  if (sol) {  // the reference's return layout, :54-60
    for (int t = 0; t < T; ++t) {
      sol[((int64_t)0 * T + t) * m + i] = X[(t * 4 + 0) * LS] + ox;
      sol[((int64_t)1 * T + t) * m + i] = X[(t * 4 + 1) * LS] + oy;
      sol[((int64_t)2 * T + t) * m + i] = X[(t * 4 + 2) * LS];
      sol[((int64_t)3 * T + t) * m + i] = X[(t * 4 + 3) * LS];
    }
    for (int t = 0; t < N; ++t) {
      sol[((int64_t)4 * T + t) * m + i] = U[(t * 2 + 0) * LS];
      sol[((int64_t)4 * T + N + t) * m + i] = U[(t * 2 + 1) * LS];
    }
  }
  if (u0) {  // (a_0, delta_0): what the caller feeds update(), :376
    u0[0 * m + i] = U[1 * LS];
    u0[1 * m + i] = U[0 * LS];
  }
  if (cost) cost[i] = J;
  if (status) status[i] = st;
  if (iters) iters[i] = it_count;
}

static void mpc_fill(MpcP* p, const crb_mpc_params* prm) {
  p->dt = prm->dt;
  p->inv_dt = 1.0f / prm->dt;
  p->inv_wb = 1.0f / prm->wb;
  p->max_steer = prm->max_steer;
  p->max_accel = prm->max_accel;
  p->max_speed = prm->max_speed;
  p->min_speed = prm->min_speed;
  p->w_a = prm->w_a; p->w_delta = prm->w_delta; p->w_da = prm->w_da; p->w_ddelta = prm->w_ddelta;
  p->wq[0] = prm->w_x; p->wq[1] = prm->w_y; p->wq[2] = prm->w_yaw; p->wq[3] = prm->w_v;
  p->max_iter = prm->max_iter;
  p->du_th = prm->du_th;
  p->max_ls = prm->max_ls;
  p->j_tol = prm->j_tol;
}

// Which solver kernel: 1 (default) = resident-slot task kernel (crb_mpc_tasks.cu), 0 = the first-generation
// thread-per-problem kernel below (CRB_MPC_VARIANT=0; kept for A/B and as the specification of the mapping
// the task kernel replaced).  Both produce the same bits.
static int mpc_variant() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("CRB_MPC_VARIANT");
    v = e ? atoi(e) : 1;
    if (v != 0) v = 1;
  }
  return v;
}

// solver scratch in floats for `count` problems
static size_t mpc_scratch_floats(crb_ctx* ctx, int T, int64_t count) {
  if (mpc_variant() == 1) return (crb_mpc_tasks_scratch_bytes(ctx->sm_count, T, count) + 3) / 4;
  const size_t ctas = (size_t)((count + MPC_BLOCK - 1) / MPC_BLOCK);  // whole CTAs
  return ctas * (size_t)mpc_ws_items(T) * MPC_BLOCK;
}

// inputs x0/xref/u_init have leading dimension ld (>= count); outputs ld_out
static int mpc_launch(crb_ctx* ctx, cudaStream_t st, int64_t count, int64_t ld, int T,
                      const float* x0, const float* xref, const float* u_init, float* scratch,
                      int64_t ld_out, float* sol, float* u0, float* cost, int32_t* status,
                      int32_t* iters, const crb_mpc_params* prm, const int32_t* hint = nullptr) {
  MpcP p;
  mpc_fill(&p, prm);
  if (mpc_variant() == 1)
    return crb_mpc_tasks_launch(ctx, st, count, ld, T, x0, xref, u_init, scratch, ld_out, sol, u0, cost,
                                status, iters, p, hint);
  // Experiment kept for A/B (CRB_MPC_L2=1): an L2 persisting access-policy window over the solver
  // workspace.  OFF by default: the set-aside shrinks the normal L2 and a workspace several times the L2's
  // size thrashes it.
  static int l2_mode = -1;
  static size_t l2_max_window = 0, l2_persist = 0;
  if (l2_mode < 0) {
    const char* e = getenv("CRB_MPC_L2");
    l2_mode = e ? atoi(e) : 0;
    if (l2_mode) {
      cudaDeviceProp prop;
      if (cudaGetDeviceProperties(&prop, ctx->device) == cudaSuccess && prop.persistingL2CacheMaxSize > 0) {
        l2_persist = (size_t)prop.persistingL2CacheMaxSize;
        l2_max_window = (size_t)prop.accessPolicyMaxWindowSize;
        if (cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, l2_persist) != cudaSuccess) l2_mode = 0;
      } else {
        l2_mode = 0;
      }
      cudaGetLastError();
    }
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)crb_grid_for(count, MPC_BLOCK));
  cfg.blockDim = dim3(MPC_BLOCK);
  cfg.stream = st;
  // A/B knob: CRB_MPC_CTAS_PER_SM=k (1..3) caps residency with dummy dynamic shared memory so that the
  // in-flight working set (k * 128 problems * 2.3 KB per SM) fits in L2.
  static int smem_cap = -1;
  if (smem_cap < 0) {
    const char* e = getenv("CRB_MPC_CTAS_PER_SM");
    const int k = e ? atoi(e) : 0;
    smem_cap = (k >= 1 && k <= 3) ? (int)((227 * 1024) / k - 2048) : 0;
  }
  if (smem_cap > 0 && !ctx->mpc_v0_attr_set) {  // per context: the attribute belongs to the device
    cudaFuncSetAttribute(crb_mpc_solve_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_cap);
    ctx->mpc_v0_attr_set = 1;
  }
  cfg.dynamicSmemBytes = (size_t)smem_cap;
  cudaLaunchAttribute attr[1];
  int nattr = 0;
  if (l2_mode) {
    size_t bytes = mpc_scratch_floats(ctx, T, count) * sizeof(float);
    if (bytes > l2_max_window) bytes = l2_max_window;
    attr[0].id = cudaLaunchAttributeAccessPolicyWindow;
    attr[0].val.accessPolicyWindow.base_ptr = scratch;
    attr[0].val.accessPolicyWindow.num_bytes = bytes;
    double ratio = bytes ? (double)l2_persist / (double)bytes : 0.0;
    attr[0].val.accessPolicyWindow.hitRatio = (float)(ratio > 1.0 ? 1.0 : ratio);
    attr[0].val.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    attr[0].val.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    nattr = 1;
  }
  cfg.attrs = attr;
  cfg.numAttrs = nattr;
  static int pfd = -1;   // CRB_MPC_PREFETCH = L2 prefetch distance in stages (0 off, 2, 3, 4)
  if (pfd < 0) {
    const char* e = getenv("CRB_MPC_PREFETCH");
    pfd = e ? atoi(e) : 0;
  }
  switch (pfd) {
    case 2:
      CRB_CUDA(cudaLaunchKernelEx(&cfg, crb_mpc_solve_kernel<2>, count, ld, T, x0, xref, u_init, scratch,
                                  ld_out, sol, u0, cost, status, iters, p));
      break;
    case 3:
      CRB_CUDA(cudaLaunchKernelEx(&cfg, crb_mpc_solve_kernel<3>, count, ld, T, x0, xref, u_init, scratch,
                                  ld_out, sol, u0, cost, status, iters, p));
      break;
    case 4:
      CRB_CUDA(cudaLaunchKernelEx(&cfg, crb_mpc_solve_kernel<4>, count, ld, T, x0, xref, u_init, scratch,
                                  ld_out, sol, u0, cost, status, iters, p));
      break;
    default:
      CRB_CUDA(cudaLaunchKernelEx(&cfg, crb_mpc_solve_kernel<0>, count, ld, T, x0, xref, u_init, scratch,
                                  ld_out, sol, u0, cost, status, iters, p));
  }
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

// The limits of crb.h (after crb_mpc_default_params), checked before any device work.  A NaN fails every comparison.
static int mpc_check_params(const crb_mpc_params* prm) {
  CRB_REQUIRE(prm != nullptr, "prm is NULL");
  const float f[] = {prm->dt, prm->wb, prm->max_steer, prm->max_accel, prm->max_speed, prm->min_speed,
                     prm->w_a, prm->w_delta, prm->w_da, prm->w_ddelta, prm->w_x, prm->w_y, prm->w_yaw, prm->w_v,
                     prm->du_th, prm->j_tol};
  for (float v : f) CRB_REQUIRE(isfinite(v), "every float parameter must be finite");
  CRB_REQUIRE(prm->dt > 0.0f && prm->wb > 0.0f, "dt and wb must be positive");
  // tan(max_steer) must exist; a steering bound below pi/2 also keeps update()'s tanf in crb_tanf_libm's range
  CRB_REQUIRE(prm->max_steer > 0.0f && (double)prm->max_steer < 1.57079632679489661923,
              "max_steer must be in (0, pi/2)");
  CRB_REQUIRE(prm->max_accel >= 0.0f, "max_accel must be >= 0");
  CRB_REQUIRE(prm->min_speed <= prm->max_speed, "min_speed must be <= max_speed");
  const float w[] = {prm->w_a, prm->w_delta, prm->w_da, prm->w_ddelta, prm->w_x, prm->w_y, prm->w_yaw, prm->w_v};
  for (float v : w) CRB_REQUIRE(v >= 0.0f, "cost weights must be >= 0");
  CRB_REQUIRE(prm->du_th >= 0.0f && prm->j_tol >= 0.0f, "du_th and j_tol must be >= 0");
  CRB_REQUIRE(prm->max_iter >= 0 && prm->max_ls >= 0, "max_iter / max_ls negative");
  return CRB_OK;
}

static int mpc_check(crb_ctx* ctx, int64_t n, int T, const float* x0, const float* xref,
                     const crb_mpc_params* prm) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  const int rc = mpc_check_params(prm);
  if (rc) return rc;
  CRB_REQUIRE(n >= 0, "n < 0");
  CRB_REQUIRE(T >= 2 && T <= CRB_MPC_MAX_T, "T out of range [2, CRB_MPC_MAX_T]");
  CRB_REQUIRE(n == 0 || (x0 && xref), "NULL array");
  return CRB_OK;
}

extern "C" int crb_mpc_solve_batched(crb_ctx* ctx, int64_t n, int T, const float* x0,
                                     const float* xref, const float* u_init,
                                     const crb_mpc_params* prm, float* sol, float* u0, float* cost,
                                     int32_t* status, int32_t* iters) {
  int rc = mpc_check(ctx, n, T, x0, xref, prm);
  if (rc) return rc;
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);   // ctx->device is current for this call, the caller's device is restored after it
  rc = crb_ctx_mpc_ws_reserve(ctx, mpc_scratch_floats(ctx, T, n) * sizeof(float));
  if (rc) return rc;
  return mpc_launch(ctx, ctx->stream, n, n, T, x0, xref, u_init, (float*)ctx->mpc_ws, n, sol,
                    u0, cost, status, iters, prm);
}

// The same solve with a scheduling hint per problem (device, [n]): an estimate of its work, e.g. the `iters` the
// previous solve of the same agent returned (receding-horizon MPC calls the solver every control step,
// src/model_predictive_control.cpp:372-378).  Problems with the largest hints start first, which removes most of the
// tail in which a few late-started long problems run alone (DESIGN.md 3).  Results are bit-identical to
// crb_mpc_solve_batched; hint must not alias `iters` (it is read while results are written).
extern "C" int crb_mpc_solve_batched_hinted(crb_ctx* ctx, int64_t n, int T, const float* x0, const float* xref,
                                            const float* u_init, const crb_mpc_params* prm, float* sol,
                                            float* u0, float* cost, int32_t* status, int32_t* iters,
                                            const int32_t* hint) {
  int rc = mpc_check(ctx, n, T, x0, xref, prm);
  if (rc) return rc;
  CRB_REQUIRE(hint == nullptr || hint != iters, "hint must not alias iters");
  if (n == 0) return CRB_OK;
  CRB_DEVICE_GUARD(ctx);
  rc = crb_ctx_mpc_ws_reserve(ctx, mpc_scratch_floats(ctx, T, n) * sizeof(float));
  if (rc) return rc;
  return mpc_launch(ctx, ctx->stream, n, n, T, x0, xref, u_init, (float*)ctx->mpc_ws, n, sol, u0, cost, status,
                    iters, prm, hint);
}

extern "C" int crb_mpc_solve_batched_host(crb_ctx* ctx, int64_t n, int T, const float* x0,
                                          const float* xref, const float* u_init,
                                          const crb_mpc_params* prm, float* sol, float* u0,
                                          float* cost, int32_t* status, int32_t* iters) {
  int rc = mpc_check(ctx, n, T, x0, xref, prm);
  if (rc) return rc;
  if (n == 0) return CRB_OK;
  CRB_CUDA(cudaSetDevice(ctx->device));
  const int N = T - 1;
  static int64_t chunk_pref = 0;  // CRB_MPC_CHUNK overrides the staging chunk (problems) for A/B
  if (chunk_pref == 0) {
    const char* e = getenv("CRB_MPC_CHUNK");
    // 8192 problems x CRB_N_PIPE = 8 slots: every chunk is resident at once and the first solve starts
    // after 1/8 of the upload
    chunk_pref = e ? atoll(e) : 8192;
    if (chunk_pref < 128) chunk_pref = 8192;
  }
  const int64_t chunk_cap = n < chunk_pref ? n : chunk_pref;
  const size_t nsol = (size_t)4 * T + 2 * N;
  // per slot: inputs (4 + 4T + 2N), outputs (nsol + 2 + 1 + 1 + 1), then the solver workspace
  const size_t nf = (size_t)4 + 4 * T + 2 * N + nsol + 5;
  const size_t pitch = (size_t)chunk_cap * sizeof(float);
  for (int s = 0; s < CRB_N_PIPE; ++s) {
    rc = crb_ctx_pipe_reserve(ctx, s, nf * pitch + mpc_scratch_floats(ctx, T, chunk_cap) * sizeof(float));
    if (rc) return rc;
  }
  const size_t hp = (size_t)n * sizeof(float);
  // Outputs in pinned + mapped memory are written by the kernel itself (see crb_host_mapped): problems
  // finish at different times, so the stores trickle over PCIe underneath the solve instead of queueing
  // as D2H copies behind it.  Inputs stay on the copy engine: a kernel that reads them over PCIe stalls
  // its whole (single) wave on the link first.
  float *msol = nullptr, *mu0 = nullptr, *mcost = nullptr;
  int32_t *mstat = nullptr, *mit = nullptr;
  // (only the first-generation kernel: its warps store 32 consecutive problems per instruction, whereas the task
  // kernel retires problems in completion order, i.e. as scattered 4-byte stores, which PCIe turns into one
  // transaction each)
  const bool direct_out = mpc_variant() == 0 && crb_zero_copy_enabled() && crb_host_mapped(sol, &msol) &&
                          crb_host_mapped(u0, &mu0) && crb_host_mapped(cost, &mcost) &&
                          crb_host_mapped(status, &mstat) && crb_host_mapped(iters, &mit);
  int slot = 0;
  for (int64_t i0 = 0; i0 < n; i0 += chunk_cap, slot = (slot + 1) % CRB_N_PIPE) {
    const int64_t cnt = (n - i0) < chunk_cap ? (n - i0) : chunk_cap;
    cudaStream_t st = ctx->pipe_stream[slot];
    float* dx0 = (float*)ctx->pipe_buf[slot];
    float* dxr = dx0 + 4 * chunk_cap;
    float* dui = dxr + (size_t)4 * T * chunk_cap;
    float* dsol = dui + (size_t)2 * N * chunk_cap;
    float* du0 = dsol + nsol * chunk_cap;
    float* dcost = du0 + 2 * chunk_cap;
    int32_t* dstat = (int32_t*)(dcost + chunk_cap);
    int32_t* dit = dstat + chunk_cap;
    float* scratch = (float*)(dit + chunk_cap);
    const size_t w = (size_t)cnt * sizeof(float);
    CRB_CUDA(crb_copy_rows(dx0, pitch, x0 + i0, hp, w, 4, cudaMemcpyHostToDevice, st));
    CRB_CUDA(crb_copy_rows(dxr, pitch, xref + i0, hp, w, (size_t)4 * T, cudaMemcpyHostToDevice,
                               st));
    if (u_init)
      CRB_CUDA(crb_copy_rows(dui, pitch, u_init + i0, hp, w, (size_t)2 * N,
                                 cudaMemcpyHostToDevice, st));
    if (direct_out) {  // results stored straight into the caller's pinned arrays (leading dimension n)
      rc = mpc_launch(ctx, st, cnt, chunk_cap, T, dx0, dxr, u_init ? dui : nullptr, scratch, n,
                      sol ? msol + i0 : nullptr, u0 ? mu0 + i0 : nullptr, cost ? mcost + i0 : nullptr,
                      status ? mstat + i0 : nullptr, iters ? mit + i0 : nullptr, prm);
      if (rc) return rc;
      continue;
    }
    rc = mpc_launch(ctx, st, cnt, chunk_cap, T, dx0, dxr, u_init ? dui : nullptr, scratch,
                    chunk_cap, sol ? dsol : nullptr, u0 ? du0 : nullptr, cost ? dcost : nullptr,
                    status ? dstat : nullptr, iters ? dit : nullptr, prm);
    if (rc) return rc;
    if (sol)
      CRB_CUDA(crb_copy_rows(sol + i0, hp, dsol, pitch, w, nsol, cudaMemcpyDeviceToHost, st));
    if (u0) CRB_CUDA(crb_copy_rows(u0 + i0, hp, du0, pitch, w, 2, cudaMemcpyDeviceToHost, st));
    if (cost) CRB_CUDA(cudaMemcpyAsync(cost + i0, dcost, w, cudaMemcpyDeviceToHost, st));
    if (status) CRB_CUDA(cudaMemcpyAsync(status + i0, dstat, w, cudaMemcpyDeviceToHost, st));
    if (iters) CRB_CUDA(cudaMemcpyAsync(iters + i0, dit, w, cudaMemcpyDeviceToHost, st));
  }
  for (int s = 0; s < CRB_N_PIPE; ++s) CRB_CUDA(cudaStreamSynchronize(ctx->pipe_stream[s]));
  return CRB_OK;
}

// ---- update(): src/model_predictive_control.cpp:69-81 ------------------------------------------------
// The step itself is crb_plant_step (crb_plant.cuh).
// The constants come from crb_mpc_params (floats).  A parameter that equals the reference's macro rounded to
// float is taken as the macro's own double value (so the defaults reproduce the reference bit for bit);
// any other value is promoted from float.  The solver, the plant step and the xref lookup therefore always
// use the same model.
static double mpc_promote(float v, double ref) { return v == (float)ref ? ref : (double)v; }
static PlantC mpc_plant_constants(const crb_mpc_params* prm) {
  PlantC c;
  c.max_steer = mpc_promote(prm->max_steer, 45.0 / 180 * 3.14159265358979323846);
  c.dt = mpc_promote(prm->dt, 0.2);
  c.wb = mpc_promote(prm->wb, 2.5);
  c.max_speed = mpc_promote(prm->max_speed, 55.0 / 3.6);
  c.min_speed = mpc_promote(prm->min_speed, -20.0 / 3.6);
  return c;
}

__global__ void __launch_bounds__(256)
crb_mpc_plant_update_kernel(int64_t n, float* __restrict__ state, const float* __restrict__ u0,
                            const PlantC k) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float x = state[i], y = state[n + i], yaw = state[2 * n + i], v = state[3 * n + i];
  crb_plant_step(x, y, yaw, v, u0[i], u0[n + i], k);
  state[i] = x; state[n + i] = y; state[2 * n + i] = yaw; state[3 * n + i] = v;
}

extern "C" int crb_mpc_plant_update_batched(crb_ctx* ctx, int64_t n, float* state, const float* u0,
                                            const crb_mpc_params* prm) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  const int rc = mpc_check_params(prm);
  if (rc) return rc;
  CRB_REQUIRE(n >= 0, "n < 0");
  if (n == 0) return CRB_OK;
  CRB_REQUIRE(state && u0, "NULL array");
  CRB_DEVICE_GUARD(ctx);   // ctx->device is current for this call, the caller's device is restored after it
  crb_mpc_plant_update_kernel<<<crb_grid_for(n, 256), 256, 0, ctx->stream>>>(n, state, u0,
                                                                             mpc_plant_constants(prm));
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

// ---- calc_ref_trajectory :130-170 with calc_nearest_index :107-127 -------------------------------------
// Agent i against the course cx .. sp of ncourse points; both lookup kernels run it.  The search window and the end
// clamp never leave [0, ncourse): an index at or past 2^31 (a target_ind below -9) ends the window, as one at or past
// ncourse does, and ind + dind is compared in 64 bits, so a sum past INT_MAX clamps to the last point.
__device__ __forceinline__ void mpc_ref_traj_agent(int64_t i, int64_t n, int T, float sx, float sy, float sv,
                                                   const float* __restrict__ cx, const float* __restrict__ cy,
                                                   const float* __restrict__ cyaw, const float* __restrict__ sp,
                                                   int ncourse, float dl, int32_t* __restrict__ target_ind,
                                                   float* __restrict__ xref, const double DT) {
  const int pind = target_ind[i];
  // calc_nearest_index: float-typed index (:109), strict '<' keeps the first minimum (:115)
  float mind = 3.402823466e+38f;
  float find = 0;
  for (unsigned int j = (unsigned int)pind; j < (unsigned int)pind + 10u; ++j) {
    if (j >= (unsigned int)ncourse) break;
    const float idx = cx[j] - sx;
    const float idy = cy[j] - sy;
    const float d_e = idx * idx + idy * idy;
    if (d_e < mind) { mind = d_e; find = (float)j; }
  }
  int ind = (int)find;
  if (pind >= ind) ind = pind;  // :139
  float travel = 0.0f;
  for (int t = 0; t < T; ++t) {
    travel = (float)((double)travel + (double)fabsf(sv) * DT);  // :149
    const int dind = (int)roundf(travel / dl);                  // :150
    const int j = (int64_t)ind + dind < ncourse ? ind + dind : ncourse - 1;
    xref[((int64_t)t * 4 + 0) * n + i] = cx[j];
    xref[((int64_t)t * 4 + 1) * n + i] = cy[j];
    xref[((int64_t)t * 4 + 2) * n + i] = cyaw[j];
    xref[((int64_t)t * 4 + 3) * n + i] = sp[j];
  }
  target_ind[i] = ind;  // :169
}

__global__ void __launch_bounds__(256)
crb_mpc_ref_traj_kernel(int64_t n, int T, const float* __restrict__ state,
                        const float* __restrict__ cx, const float* __restrict__ cy,
                        const float* __restrict__ cyaw, const float* __restrict__ sp, int ncourse,
                        float dl, int32_t* __restrict__ target_ind, float* __restrict__ xref,
                        const double DT) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  mpc_ref_traj_agent(i, n, T, state[i], state[n + i], state[3 * n + i], cx, cy, cyaw, sp, ncourse, dl, target_ind,
                     xref, DT);
}

// The lookup with a course per agent: the agent's course reference is checked before any course data is read
// (course_of[i] in [0, n_courses), 0 <= course_off[c] < course_off[c + 1] <= npts, a length that fits in int); a bad
// one gives NaN xref, leaves target_ind and sets CRB_MPC_REF_BAD_COURSE.  One thread per agent: the window is 10
// points and the horizon at most CRB_MPC_MAX_T.
__global__ void __launch_bounds__(256)
crb_mpc_lookup_many_kernel(int64_t n, int T, const float* __restrict__ state, const float* __restrict__ cx,
                           const float* __restrict__ cy, const float* __restrict__ cyaw,
                           const float* __restrict__ sp, const int64_t* __restrict__ course_off, int32_t n_courses,
                           int64_t npts, const int32_t* __restrict__ course_of, float dl,
                           int32_t* __restrict__ target_ind, float* __restrict__ xref, int32_t* __restrict__ status,
                           const double DT) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t c = course_of[i];
  int64_t a = 0, b = 0;
  if (c >= 0 && c < n_courses) { a = course_off[c]; b = course_off[c + 1]; }
  if (c < 0 || c >= n_courses || a < 0 || a >= b || b > npts || b - a > 0x7fffffff) {
    const float q = __int_as_float(0x7fffffff);
    for (int f = 0; f < 4 * T; ++f) xref[(int64_t)f * n + i] = q;
    if (status) status[i] = CRB_MPC_REF_BAD_COURSE;
    return;
  }
  mpc_ref_traj_agent(i, n, T, state[i], state[n + i], state[3 * n + i], cx + a, cy + a, cyaw + a, sp + a, (int)(b - a),
                     dl, target_ind, xref, DT);
  if (status) status[i] = CRB_MPC_REF_OK;
}

static int mpc_check_lookup(int64_t n, int T, float dl, const crb_mpc_params* prm) {
  CRB_REQUIRE(n >= 0 && T >= 1 && T <= CRB_MPC_MAX_T, "n < 0 or T out of range");
  CRB_REQUIRE(dl > 0.0f, "dl <= 0");
  // the lookup uses only dt
  CRB_REQUIRE(prm != nullptr && isfinite(prm->dt) && prm->dt > 0.0f, "prm is NULL or dt not finite and > 0");
  return CRB_OK;
}

extern "C" int crb_mpc_calc_ref_trajectory_batched(crb_ctx* ctx, int64_t n, int T,
                                                   const float* state, const float* cx,
                                                   const float* cy, const float* cyaw,
                                                   const float* sp, int32_t ncourse, float dl,
                                                   int32_t* target_ind, float* xref,
                                                   const crb_mpc_params* prm) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(ncourse >= 1, "empty course");
  const int rc = mpc_check_lookup(n, T, dl, prm);
  if (rc) return rc;
  if (n == 0) return CRB_OK;
  CRB_REQUIRE(state && cx && cy && cyaw && sp && target_ind && xref, "NULL array");
  CRB_DEVICE_GUARD(ctx);   // ctx->device is current for this call, the caller's device is restored after it
  crb_mpc_ref_traj_kernel<<<crb_grid_for(n, 256), 256, 0, ctx->stream>>>(
      n, T, state, cx, cy, cyaw, sp, ncourse, dl, target_ind, xref, mpc_plant_constants(prm).dt);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}

extern "C" int crb_mpc_calc_ref_trajectory_many_batched(crb_ctx* ctx, int64_t n, int T, const float* state,
                                                        const float* cx, const float* cy, const float* cyaw,
                                                        const float* sp, const int64_t* course_off,
                                                        int32_t n_courses, int64_t npts, const int32_t* course_of,
                                                        float dl, int32_t* target_ind, float* xref, int32_t* status,
                                                        const crb_mpc_params* prm) {
  CRB_REQUIRE(ctx != nullptr, "ctx is NULL");
  CRB_REQUIRE(n_courses >= 1 && npts >= 1, "n_courses and npts must be >= 1");
  const int rc = mpc_check_lookup(n, T, dl, prm);
  if (rc) return rc;
  if (n == 0) return CRB_OK;
  CRB_REQUIRE(state && cx && cy && cyaw && sp && course_off && course_of && target_ind && xref, "NULL array");
  CRB_DEVICE_GUARD(ctx);
  crb_mpc_lookup_many_kernel<<<crb_grid_for(n, 256), 256, 0, ctx->stream>>>(
      n, T, state, cx, cy, cyaw, sp, course_off, n_courses, npts, course_of, dl, target_ind, xref, status,
      mpc_plant_constants(prm).dt);
  CRB_CUDA(cudaGetLastError());
  ctx->launches++;
  return CRB_OK;
}
