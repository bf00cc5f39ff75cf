"""Writes tests/golden/lqr_track_golden.npz from the reference's own text (oracle/_ref/libref_lqrt4.so and
libref_lqrt5.so, built by `make -C oracle` where the reference tree is present): lqr_steering_control's
outputs (u, ind, pe, pth_e) for 512 vehicles on each program's demo-shaped course, and update on 512 states.

  python tests/golden/make_lqr_track_golden.py"""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import lqr_track_cases as LC  # noqa: E402
from cpprobotics_b200 import synth  # noqa: E402
from oracle._load import reference  # noqa: E402

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
N = 512


def main():
    out = {}
    state = ind = pe = pth_e = None
    for nx in (4, 5):
        L = reference(f"lqrt{nx}")
        if L is None:
            raise SystemExit("oracle/_ref not built: needs the reference tree (make -C oracle)")
        course = synth.lqr_course("demo" if nx == 4 else "demo_speed")
        if state is None:
            state, ind, pe, pth_e = synth.lqr_track_inputs(N, course, seed=0x601D)
        cx, cy, cyaw, ck, sp = course
        fr, ir = C.POINTER(C.c_float), C.POINTER(C.c_int)
        u = np.zeros((1 if nx == 4 else 2, N), np.float32)
        o_ind, o_pe, o_pth = ind.copy(), pe.copy(), pth_e.copy()
        for i in range(N):
            st = np.ascontiguousarray(state[:, i])
            e, t = C.c_float(pe[i]), C.c_float(pth_e[i])
            if nx == 4:
                L.ref_lqr_control4.restype = C.c_float
                L.ref_lqr_control4.argtypes = [f32p] * 5 + [C.c_int, ir, fr, fr]
                j = C.c_int(int(ind[i]))
                u[0, i] = L.ref_lqr_control4(st, cx, cy, cyaw, ck, cx.size, C.byref(j), C.byref(e), C.byref(t))
            else:
                L.ref_lqr_control5.restype = None
                L.ref_lqr_control5.argtypes = [f32p] * 6 + [C.c_int, fr, fr, f32p]
                L.ref_lqr_nearest5.restype = C.c_float
                L.ref_lqr_nearest5.argtypes = [f32p] * 4 + [C.c_int, ir]
                r = np.zeros(2, np.float32)
                L.ref_lqr_control5(st, cx, cy, cyaw, ck, sp, cx.size, C.byref(e), C.byref(t), r)
                u[:, i] = r
                j = C.c_int(0)
                L.ref_lqr_nearest5(st, cx, cy, cyaw, cx.size, C.byref(j))
            o_ind[i], o_pe[i], o_pth[i] = j.value, e.value, t.value
        out.update({f"course{nx}": np.stack(course), f"u{nx}": u, f"ind{nx}": o_ind, f"pe{nx}": o_pe,
                    f"pth_e{nx}": o_pth})
    out.update(state=state, ind=ind, pe=pe, pth_e=pth_e)
    st, a, delta = LC.update_cases(N, seed=0x601E)
    L = reference("lqrt4")
    L.ref_lqr_update4.restype = None
    L.ref_lqr_update4.argtypes = [f32p, C.c_float, C.c_float]
    new = st.copy()
    for i in range(N):
        s = np.ascontiguousarray(new[:, i])
        L.ref_lqr_update4(s, float(a[i]), float(delta[i]))
        new[:, i] = s
    out.update(ustate=st, ua=a, udelta=delta, unew=new)
    np.savez_compressed(os.path.join(HERE, "lqr_track_golden.npz"), **out)
    print("wrote tests/golden/lqr_track_golden.npz")


if __name__ == "__main__":
    main()
