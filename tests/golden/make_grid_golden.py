"""Writes tests/golden/grid_golden.npz from the reference's own text (oracle/_ref/libref_astar.so, libref_dijkstra.so,
built by `make -C oracle` where the reference tree is present): for each planner, the demo's obstacle map,
expansion trace and path, and 24 seeded scenarios' inputs and paths (tests/grid_cases.py).  Cells are int16.

  python tests/golden/make_grid_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import grid_cases as GC  # noqa: E402
from oracle import grid as OG  # noqa: E402

SEEDED = 24


def main():
    out = {}
    for algo, name in GC.ALGOS:
        L = GC.ref_lib(algo)
        if L is None:
            raise SystemExit("oracle/_ref not built: needs the reference tree (make -C oracle)")
        ox, oy, reso, rr, sg = GC.demo()
        r = GC.ref_run(L, *sg[:, 0], ox, oy, reso, rr)
        for k in ("map_cells", "trace", "path"):
            out[f"demo_{name}_{k}"] = r[k].astype(np.int16)
        ins, paths, plen, olen = [], [], [], []
        for s in GC.seeded_scenarios(algo, 4 * SEEDED, seed=0x601D + algo):
            ox, oy, reso, rr, sx, sy, gx, gy = s
            box = OG.box_of_obstacles(ox, oy, reso)
            m = OG.obstacle_map(ox, oy, reso, rr, box)
            st = OG.plan(algo, box, m, reso, np.float32([[sx], [sy], [gx], [gy]]))["status"][0]
            if not GC.check_ref_domain(algo, box, st):
                continue
            p = GC.ref_run(L, sx, sy, gx, gy, ox, oy, reso, rr)["path"]
            ins.append(np.concatenate([[reso, rr, sx, sy, gx, gy], ox, oy]).astype(np.float32))
            olen.append(ox.size)
            paths.append(p.astype(np.int16))
            plen.append(len(p))
            if len(ins) == SEEDED:
                break
        out[f"seeded_{name}_inputs"] = np.concatenate(ins)
        out[f"seeded_{name}_n_obs"] = np.int32(olen)
        out[f"seeded_{name}_path"] = np.concatenate(paths)
        out[f"seeded_{name}_path_len"] = np.int32(plen)
    np.savez_compressed(os.path.join(HERE, "grid_golden.npz"), **out)


if __name__ == "__main__":
    main()
