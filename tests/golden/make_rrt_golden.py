"""Writes tests/golden/rrt_golden.npz from the reference's own text (oracle/_ref/libref_rrt.so, built by
`make -C oracle -f rrt.mk` where the reference tree is present): the demo's node_list (tree, parents) and path for
goal_gen seeds 1..32, and 16 scattered maps' inputs and paths (tests/rrt_cases.py).

  python tests/golden/make_rrt_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import rrt_cases as RC  # noqa: E402
from cpprobotics_b200 import synth  # noqa: E402

DEMO_SEEDS = 32
SCATTERED = 16


def main():
    L = RC.ref_lib()
    if L is None:
        raise SystemExit("oracle/_ref not built: needs the reference tree (make -C oracle -f rrt.mk)")
    d = synth.RRT_DEMO
    prm, ob = RC.demo_prm(), synth.rrt_demo_obstacles()
    out = {}
    trees, parents, paths, nn, pl = [], [], [], [], []
    for s in range(1, DEMO_SEEDS + 1):
        r = RC.ref_run(L, prm, ob, d["sx"], d["sy"], d["gx"], d["gy"], s, prm["max_iter"] + 1)
        trees.append(r["tree"]); parents.append(r["parent"]); paths.append(r["path"])
        nn.append(len(r["parent"])); pl.append(len(r["path"]))
    out.update(demo_tree=np.concatenate(trees), demo_parent=np.concatenate(parents).astype(np.int16),
               demo_path=np.concatenate(paths), demo_n_nodes=np.int32(nn), demo_path_len=np.int32(pl))
    ins, n_ob, paths, pl = [], [], [], []
    for prm, ob, sx, sy, gx, gy, seed in RC.scattered_maps(4 * SCATTERED, seed=0x601D):
        if RC.checker_one(prm, ob, sx, sy, gx, gy, seed)["status"] != 0:
            continue
        r = RC.ref_run(L, prm, ob, sx, sy, gx, gy, seed, prm["max_iter"] + 1)
        ins.append(np.concatenate([[prm["rand_min"], prm["rand_max"], prm["expand_dis"], prm["goal_sample_rate"],
                                    sx, sy, gx, gy, np.uint32(seed).view(np.float32)], ob.reshape(-1)]).astype(np.float32))
        n_ob.append(ob.shape[0]); paths.append(r["path"]); pl.append(len(r["path"]))
        if len(ins) == SCATTERED:
            break
    out.update(scattered_inputs=np.concatenate(ins), scattered_n_ob=np.int32(n_ob),
               scattered_path=np.concatenate(paths), scattered_path_len=np.int32(pl))
    np.savez_compressed(os.path.join(HERE, "rrt_golden.npz"), **out)


if __name__ == "__main__":
    main()
