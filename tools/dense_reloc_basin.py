#!/usr/bin/env python
"""The basin of the coarse-to-fine alignment against the whole-run voxel map, which the relocalisation grid's steps
must stay inside.

Scene: the static-sweep scene of tests/test_align_reference.py (a map from 4 static sweeps, VLP-16 and HDL-64E, leaf
0.1 and 0.2, target at normals radius 2).  For every full-density held-out sweep, every offset (yaw in degrees,
translation in metres on the x-z ground plane) is applied in 8 directions (0, 45, ..., 315 deg) with both signs of
the yaw, and the sweep is aligned coarse to fine (dense_align_batch at radius 3, then 1, 30 iterations each; equal to
dense_align run by run).  A run succeeds when it converged within the alignment bars (1 cm, 0.1 deg) of the truth.
Prints one JSON line: per configuration and offset, the successes out of the runs.

    python tools/dense_reloc_basin.py [--yaw 0,0.5,1,1.5,2,2.5 --metres 0,0.1,0.2,0.25,0.3,0.35,0.5]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

import numpy as np

sys.dont_write_bytecode = True
from dense_cost import ROOT, dense_ctx, gpu_info, require_cuda  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--yaw", default="0,0.5,1,1.5,2,2.5")
    ap.add_argument("--metres", default="0,0.1,0.2,0.25,0.3,0.35,0.5")
    args = ap.parse_args()
    yaws = [float(v) for v in args.yaw.split(",")]
    metres = [float(v) for v in args.metres.split(",")]

    require_cuda("dense_reloc_basin")
    import align_reference as ar
    from loam_velodyne_b200 import synth
    from test_align_reference import BAR_DEG, BAR_M, HELD_OUT, MAP_TWISTS, lidars

    scene = synth.make_scene()
    out = {}
    for sensor, lidar in lidars().items():
        for leaf in (0.1, 0.2):
            c, _ = dense_ctx([ar.static_sweep(scene, lidar, tw, seed=k)[1] for k, tw in enumerate(MAP_TWISTS)], leaf)
            c.dense_target_build(None, 2)
            ok = {(y, m): 0 for y in yaws for m in metres}
            runs = {(y, m): 0 for y in yaws for m in metres}
            for h, truth in enumerate(HELD_OUT):
                pts = ar.static_sweep(scene, lidar, truth.astype(np.float64), seed=100 + h)[0]
                init, cells = [], []
                for y in yaws:
                    for m in metres:
                        for d in range(8):
                            a = math.radians(45.0 * d)
                            for sign in (1.0, -1.0):
                                init.append(truth + np.array([0, sign * math.radians(y), 0, m * math.cos(a), 0,
                                                              m * math.sin(a)], np.float32))
                                cells.append((y, m))
                init = np.array(init, np.float32)
                coarse, _ = c.dense_align_batch(pts, init, 3, 30)
                fine, infos = c.dense_align_batch(pts, coarse, 1, 30)
                for j, cell in enumerate(cells):
                    e_m, e_deg = ar.twist_error(fine[j], truth)
                    runs[cell] += 1
                    ok[cell] += int(infos[j]["converged"] and e_m <= BAR_M and e_deg <= BAR_DEG)
            c.close()
            out[f"{sensor}_leaf{leaf}"] = {f"{y}deg_{m}m": f"{ok[(y, m)]}/{runs[(y, m)]}" for y in yaws for m in metres}
    print(json.dumps({"basin": out, "gpu": gpu_info()}))


if __name__ == "__main__":
    main()
