// oracle/shim/ref_wrap_lqrt.cpp — C entry points around the LQR programs' own calc_nearest_index,
// lqr_steering_control and update.  The reference source file is #included from where it lies (REF_SRC, set by
// oracle/Makefile) with main() renamed; nothing of it is copied into this repository.  WHICH selects the program:
// 4 src/lqr_steer_control.cpp, 5 src/lqr_speed_steer_control.cpp.  st is (x, y, yaw, v).
#define main crb_reference_main
#include REF_SRC
#undef main

extern "C" {
#if WHICH == 4
// calc_nearest_index :55-73, lqr_steering_control :98-133, update :136-146
float ref_lqr_nearest4(const float* st, const float* cx, const float* cy, const float* cyaw, int n, int* ind) {
  State s(st[0], st[1], st[2], st[3]);
  return calc_nearest_index(s, Vec_f(cx, cx + n), Vec_f(cy, cy + n), Vec_f(cyaw, cyaw + n), *ind);
}
float ref_lqr_control4(const float* st, const float* cx, const float* cy, const float* cyaw, const float* ck, int n,
                       int* ind, float* pe, float* pth_e) {
  State s(st[0], st[1], st[2], st[3]);
  return lqr_steering_control(s, Vec_f(cx, cx + n), Vec_f(cy, cy + n), Vec_f(cyaw, cyaw + n), Vec_f(ck, ck + n), *ind,
                              *pe, *pth_e);
}
void ref_lqr_update4(float* st, float a, float delta) {
  State s(st[0], st[1], st[2], st[3]);
  update(s, a, delta);
  st[0] = s.x; st[1] = s.y; st[2] = s.yaw; st[3] = s.v;
}
#elif WHICH == 5
// calc_nearest_index :65-83, lqr_steering_control :108-151 (out2 = {ai, delta}), update :154-164
float ref_lqr_nearest5(const float* st, const float* cx, const float* cy, const float* cyaw, int n, int* ind) {
  State s(st[0], st[1], st[2], st[3]);
  return calc_nearest_index(s, Vec_f(cx, cx + n), Vec_f(cy, cy + n), Vec_f(cyaw, cyaw + n), *ind);
}
void ref_lqr_control5(const float* st, const float* cx, const float* cy, const float* cyaw, const float* ck,
                      const float* sp, int n, float* pe, float* pth_e, float* out2) {
  State s(st[0], st[1], st[2], st[3]);
  Vec_f r = lqr_steering_control(s, Vec_f(cx, cx + n), Vec_f(cy, cy + n), Vec_f(cyaw, cyaw + n), Vec_f(ck, ck + n),
                                 Vec_f(sp, sp + n), *pe, *pth_e);
  out2[0] = r[0];
  out2[1] = r[1];
}
void ref_lqr_update5(float* st, float a, float delta) {
  State s(st[0], st[1], st[2], st[3]);
  update(s, a, delta);
  st[0] = s.x; st[1] = s.y; st[2] = s.yaw; st[3] = s.v;
}
#endif
}
