// oracle/shim/ref_wrap.cpp — C entry points around the reference's own functions.  The reference source
// file is #included from where it lies (REF_SRC, set by oracle/Makefile) with main() renamed; nothing of it
// is copied into this repository.  WHICH selects the program: 1 EKF, 2 PF, 3 MPC.
#define main crb_reference_main
#include REF_SRC
#undef main

extern "C" {
#if WHICH == 1
void ref_motion_model(const float* x, const float* u, float* out) {
  Eigen::Vector4f xv; Eigen::Vector2f uv;
  for (int i = 0; i < 4; ++i) xv(i) = x[i];
  uv(0) = u[0]; uv(1) = u[1];
  Eigen::Vector4f r = motion_model(xv, uv);
  for (int i = 0; i < 4; ++i) out[i] = r(i);
}
void ref_jacobF(const float* x, const float* u, float* out16) {
  Eigen::Vector4f xv; Eigen::Vector2f uv;
  for (int i = 0; i < 4; ++i) xv(i) = x[i];
  uv(0) = u[0]; uv(1) = u[1];
  Eigen::Matrix4f r = jacobF(xv, uv);
  for (int i = 0; i < 16; ++i) out16[i] = r.d[i];
}
void ref_ekf_estimation(float* x, float* P, const float* z, const float* u, const float* Q, const float* R) {
  Eigen::Vector4f xe; Eigen::Matrix4f Pe, Qm; Eigen::Vector2f zv, uv; Eigen::Matrix2f Rm;
  for (int i = 0; i < 4; ++i) xe(i) = x[i];
  for (int i = 0; i < 16; ++i) { Pe.d[i] = P[i]; Qm.d[i] = Q[i]; }
  for (int i = 0; i < 4; ++i) Rm.d[i] = R[i];
  zv(0) = z[0]; zv(1) = z[1]; uv(0) = u[0]; uv(1) = u[1];
  ekf_estimation(xe, Pe, zv, uv, Qm, Rm);
  for (int i = 0; i < 4; ++i) x[i] = xe(i);
  for (int i = 0; i < 16; ++i) P[i] = Pe.d[i];
}
#elif WHICH == 2
float ref_gauss_likelihood(float x, float sigma) { return gauss_likelihood(x, sigma); }
int ref_pf_np(void) { return NP; }
// px 4xNP column-major, pw NP; z rows (range, lx, ly); the generator is seeded here and passed BY VALUE
// exactly like main() does (:270); draws[2*NP] returns the normals the loop consumed, in order.
void ref_pf_localization(float* px, float* pw, float* xEst, float* PEst, const float* z, int nz,
                         const float* u, const float* rsim, float Q, unsigned seed, double* draws) {
  Eigen::Matrix<float, 4, NP> pxm; Eigen::Matrix<float, NP, 1> pwm;
  for (int i = 0; i < 4 * NP; ++i) pxm.d[i] = px[i];
  for (int i = 0; i < NP; ++i) pwm.d[i] = pw[i];
  std::vector<Eigen::RowVector3f> zs(nz);
  for (int i = 0; i < nz; ++i) for (int k = 0; k < 3; ++k) zs[i](k) = z[3 * i + k];
  Eigen::Vector2f uv; uv(0) = u[0]; uv(1) = u[1];
  Eigen::Matrix2f Rsim = Eigen::Matrix2f::Identity();
  Rsim(0, 0) = rsim[0]; Rsim(1, 1) = rsim[1];
  Eigen::Vector4f xe = Eigen::Vector4f::Zero(); Eigen::Matrix4f Pe = Eigen::Matrix4f::Zero();
  std::mt19937 gen{seed};
  std::normal_distribution<> gaussian_d{0, 1};
  pf_localization(pxm, pwm, xe, Pe, zs, uv, Rsim, Q, gen, gaussian_d);
  std::mt19937 gen2{seed};
  std::normal_distribution<> d2{0, 1};
  for (int i = 0; i < 2 * NP; ++i) draws[i] = d2(gen2);
  for (int i = 0; i < 4 * NP; ++i) px[i] = pxm.d[i];
  for (int i = 0; i < NP; ++i) pw[i] = pwm.d[i];
  for (int i = 0; i < 4; ++i) xEst[i] = xe(i);
  for (int i = 0; i < 16; ++i) PEst[i] = Pe.d[i];
}
// resampling() :120-148 with a seeded generator passed BY VALUE like main() does (:271); draws[NP] returns the
// uniforms it consumed (only meaningful when it resampled).  Returns 1 if the weights were reset to 1/NP.
int ref_resampling(float* px, float* pw, unsigned seed, double* draws) {
  Eigen::Matrix<float, 4, NP> pxm; Eigen::Matrix<float, NP, 1> pwm;
  for (int i = 0; i < 4 * NP; ++i) pxm.d[i] = px[i];
  for (int i = 0; i < NP; ++i) pwm.d[i] = pw[i];
  std::mt19937 gen2{seed};
  std::uniform_real_distribution<> uni_d{1.0, 2.0};
  float before = pwm(0);
  resampling(pxm, pwm, gen2, uni_d);
  std::mt19937 g3{seed};
  std::uniform_real_distribution<> u3{1.0, 2.0};
  for (int i = 0; i < NP; ++i) draws[i] = u3(g3);
  int did = 0;
  for (int i = 0; i < NP; ++i) if (pwm(i) != pw[i]) did = 1;
  (void)before;
  for (int i = 0; i < 4 * NP; ++i) px[i] = pxm.d[i];
  for (int i = 0; i < NP; ++i) pw[i] = pwm.d[i];
  return did;
}
#elif WHICH == 3
int ref_mpc_T(void) { return T; }
void ref_update(float* st, float a, float delta) {
  State s(st[0], st[1], st[2], st[3]);
  update(s, a, delta);
  st[0] = s.x; st[1] = s.y; st[2] = s.yaw; st[3] = s.v;
}
int ref_calc_nearest_index(const float* st, const float* cx, const float* cy, const float* cyaw, int n, int pind) {
  State s(st[0], st[1], st[2], st[3]);
  return calc_nearest_index(s, Vec_f(cx, cx + n), Vec_f(cy, cy + n), Vec_f(cyaw, cyaw + n), pind);
}
void ref_calc_ref_trajectory(const float* st, const float* cx, const float* cy, const float* cyaw,
                             const float* sp, int n, float dl, int* target_ind, float* xref /*4xT col-major*/) {
  State s(st[0], st[1], st[2], st[3]);
  M_XREF xr;
  calc_ref_trajectory(s, Vec_f(cx, cx + n), Vec_f(cy, cy + n), Vec_f(cyaw, cyaw + n), Vec_f(n, 0.0f),
                      Vec_f(sp, sp + n), dl, *target_ind, xr);
  for (int i = 0; i < NX * T; ++i) xref[i] = xr.d[i];
}
// fg[0] and the constraint residuals of FG_EVAL::operator() (:199-252) at a given point, in double.
// vars in the reference's layout (:54-60); fg has 1 + 4T entries.
void ref_fg_eval(const float* xref /*4xT col-major*/, const double* vars, double* fg) {
  M_XREF xr;
  for (int i = 0; i < NX * T; ++i) xr.d[i] = xref[i];
  FG_EVAL f(xr);
  FG_EVAL::ADvector fgv(1 + 4 * T), v(4 * T + 2 * (T - 1));
  for (size_t i = 0; i < v.size(); ++i) v[i] = vars[i];
  f(fgv, v);
  for (size_t i = 0; i < fgv.size(); ++i) fg[i] = CppAD::Value(fgv[i]);
}
#elif WHICH == 4
// src/lqr_steer_control.cpp: solve_DARE :75-90, dlqr :92-96 (4 states, 1 input, scalar R)
void ref_dlqr4(const float* A, const float* B, const float* Q, float R, float* K, float* X) {
  Eigen::Matrix4f Am, Qm; Eigen::Vector4f Bm;
  for (int i = 0; i < 16; ++i) { Am.d[i] = A[i]; Qm.d[i] = Q[i]; }
  for (int i = 0; i < 4; ++i) Bm(i) = B[i];
  Eigen::Matrix4f Xm = solve_DARE(Am, Bm, Qm, R);
  Eigen::RowVector4f Km = dlqr(Am, Bm, Qm, R);
  for (int i = 0; i < 4; ++i) K[i] = Km(i);
  for (int i = 0; i < 16; ++i) X[i] = Xm.d[i];
}
#elif WHICH == 5
// src/lqr_speed_steer_control.cpp: solve_DARE :85-100, dlqr :102-106 (5 states, 2 inputs)
void ref_dlqr5(const float* A, const float* B, const float* Q, const float* R, float* K, float* X) {
  Matrix5f Am, Qm; Matrix52f Bm; Eigen::Matrix2f Rm;
  for (int i = 0; i < 25; ++i) { Am.d[i] = A[i]; Qm.d[i] = Q[i]; }
  for (int i = 0; i < 10; ++i) Bm.d[i] = B[i];
  for (int i = 0; i < 4; ++i) Rm.d[i] = R[i];
  Matrix5f Xm = solve_DARE(Am, Bm, Qm, Rm);
  Matrix25f Km = dlqr(Am, Bm, Qm, Rm);
  for (int i = 0; i < 10; ++i) K[i] = Km.d[i];
  for (int i = 0; i < 25; ++i) X[i] = Xm.d[i];
}
#endif
}
