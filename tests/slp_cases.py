"""Inputs and reference calls for tests/test_slp.py and tests/golden/make_slp_golden.py: seeded sampler queries,
the corner cases of the samplers and the search, and the reference's own functions (oracle/_ref/libref_slp.so) in
the libcrb layout."""
import ctypes as C
import os

import numpy as np

from cpprobotics_b200 import synth
from oracle import slp as OS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLE_CSV = os.path.join(ROOT, "tests", "golden", "lookuptable.csv")
REF = os.path.join(ROOT, "oracle", "_ref", "libref_slp.so")


def table():
    from cpprobotics_b200 import slp_load_table
    return slp_load_table(TABLE_CSV)


def sampler_of(fields, **over):
    f = dict(fields, **over)
    return OS.sampler(f["kind"], f["nxy"], f["nh"], f["ns"], f["d"])


def ref_lib():
    return C.CDLL(REF) if os.path.exists(REF) else None


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def ref_sample(L, s, qp):
    """The reference's sampler per query, in crb_slp_sample_states_batched's layout: (target [3, n*S], n_states)."""
    qp = np.ascontiguousarray(qp, np.float32)
    n = qp.shape[1]
    S = OS.states_per_query(s)
    target = np.full((3, n * S), np.nan, np.float32)
    cnt = np.zeros(n, np.int32)
    buf = np.empty(3 * max(S, 1), np.float32)
    F = C.c_float
    for q in range(n):
        v = [float(x) for x in qp[:, q]]
        if s.kind == OS.UNIFORM:
            k = L.ref_slp_uniform(s.nxy, s.nh, s.d, F(v[0]), F(v[1]), F(v[2]), F(v[3]), _vp(buf), S)
        elif s.kind == OS.BIASED:
            k = L.ref_slp_biased(F(v[0]), s.ns, s.nxy, s.nh, s.d, F(v[1]), F(v[2]), F(v[3]), F(v[4]), _vp(buf), S)
        else:
            k = L.ref_slp_lane(F(v[0]), F(v[1]), F(v[2]), F(v[3]), F(v[4]), s.nxy, _vp(buf), S)
        assert 0 <= k <= S, (q, k, S)
        cnt[q] = k
        target[:, q * S:q * S + k] = buf[:3 * k].reshape(k, 3).T
    return target, cnt


def ref_search(L, target, tb):
    """search_nearest_one_from_lookuptable per target: param [4, n] (steering[0] = 0, as the function returns it)."""
    t = np.ascontiguousarray(np.asarray(target, np.float32).T)
    tb = np.ascontiguousarray(tb, np.float32)
    out = np.empty((t.shape[0], 4), np.float32)
    L.ref_slp_search(t.shape[0], _vp(t), _vp(tb), tb.shape[0], _vp(out))
    return np.ascontiguousarray(out.T)


def ref_generate_path(L, target, tb, k0, max_pts):
    """generate_path(states, table, k0): (traj [3*max_pts, n] NaN past each trajectory, traj_len [n])."""
    t = np.ascontiguousarray(np.asarray(target, np.float32).T)
    tb = np.ascontiguousarray(tb, np.float32)
    n = t.shape[0]
    traj = np.full((n, max_pts, 3), np.nan, np.float32)
    ln = np.zeros(n, np.int32)
    L.ref_slp_generate_path(n, _vp(t), _vp(tb), tb.shape[0], C.c_float(k0), _vp(traj), max_pts, _vp(ln))
    return np.ascontiguousarray(traj.reshape(n, 3 * max_pts).T), ln


def ref_demo(L, which, tb, max_pts, cap=256):
    traj = np.full((cap, max_pts, 3), np.nan, np.float32)
    ln = np.zeros(cap, np.int32)
    tb = np.ascontiguousarray(tb, np.float32)
    n = L.ref_slp_demo(which, _vp(tb), tb.shape[0], _vp(traj), max_pts, _vp(ln), cap)
    return np.ascontiguousarray(traj[:n].reshape(n, 3 * max_pts).T), ln[:n]


def ref_read_csv(L, path, cap=1 << 16):
    out = np.empty((cap, 6), np.float32)
    k = L.ref_slp_read_csv(str(path).encode(), _vp(out), cap)
    return None if k < 0 else out[:k].copy()


def demo(kind):
    """The demo's sampler and its one query."""
    fields, qp = synth.slp_inputs(1, kind)
    return sampler_of(fields), qp


def sampler_sets():
    """Samplers the reference defines, beyond the demo's integers: (name, sampler, qp) with 200 seeded queries."""
    sets = []
    for kind, name in ((OS.UNIFORM, "uniform"), (OS.BIASED, "biased"), (OS.LANE, "lane")):
        fields, qp = synth.slp_inputs(200, kind, seed=0x5A + kind)
        if kind != OS.LANE:
            sets.append((f"{name}_nh1", sampler_of(fields, nh=1), qp))            # (p_max - p_min) / 2.0 + a
            sets.append((f"{name}_nh7_d-3", sampler_of(fields, nh=7, d=-3), qp))
        sets.append((f"{name}_nxy2", sampler_of(fields, nxy=2), qp))
        sets.append((f"{name}_nxy1", sampler_of(fields, nxy=1), qp))                # 0 / 0: NaN angles
    fields, qp = synth.slp_inputs(200, OS.BIASED, seed=0x77)
    for ns in (0, 1, 2, 3):                                                           # ns <= 1: no samples at all
        sets.append((f"biased_ns{ns}", sampler_of(fields, ns=ns), qp))
    sets.append(("biased_duplicates", sampler_of(fields, ns=7, nxy=40), qp))          # the scan repeats samples
    sets.append(("biased_dense", sampler_of(fields, ns=1000, nxy=64, nh=3), qp))
    return sets


def search_sets():
    """Lookup-table corner cases: (name, target [3, n], table [rows, 6])."""
    sets = []
    tb = table()
    # targets exactly between two rows (the first wins), and on a row
    t = np.stack([(tb[3, :3] + tb[5, :3]) / 2, tb[7, :3], tb[0, :3]], axis=1).astype(np.float32)
    two = np.float32([[2, 0, 0, 0, 0.1, 0.2], [0, 0, 0, 0, 0.3, 0.4]])
    sets.append(("equidistant", np.float32([[1.0], [0.0], [0.0]]), two))
    sets.append(("table_points", t, tb))
    # distinct squares whose float roots are equal: the first row is farther in squares, but its root ties
    a, e = _equal_root_rows()
    eq = np.float32([[a, 0, e, 0, 1.0, 2.0], [a, 0, 0, 0, 3.0, 4.0]])
    sets.append(("equal_roots", np.float32([[0.0], [0.0], [0.0]]), eq))
    # a NaN row and an inf row never win; a one-row table
    bad = tb.copy()
    bad[0, 0] = np.nan
    bad[1, 2] = np.inf
    sets.append(("nan_row", np.ascontiguousarray(tb[:4, :3].T), bad))
    sets.append(("one_row", np.float32([[3.0, -1.0], [1.0, 2.0], [0.2, 0.0]]), tb[10:11].copy()))
    return sets


def _equal_root_rows():
    """(x, e): seen from the origin, a row at (x, 0, yaw e) has the larger float square x*x + e*e, a row at (x, 0, 0)
    the smaller x*x, and sqrtf rounds both to the same root."""
    f = np.float32
    x = f(5.0)
    for k in range(1, 4096):
        e = f(k * 2.0 ** -14)
        big, small = f(f(x * x) + f(e * e)), f(x * x)
        if big != small and np.sqrt(big) == np.sqrt(small):
            return float(x), float(e)
    raise AssertionError("no equal-root pair")
