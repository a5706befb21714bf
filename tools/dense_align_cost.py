#!/usr/bin/env python
"""What aligning a sweep against the whole-run voxel map costs.

Workload: the replayed hdl64_1m map (tools/dense_cost.py), --sweeps sweeps at --leaf.  Reported, with the card's name
and power limit read in the same run:
  * the target build (dense_target_build at radius 2): GPU time of its kernels (CUDA-event profiling, family "dense")
    and host time, over --reps builds after one warm-up;
  * one iteration (dense_align_iterate) of a 131 k-point sweep at search radius 1, 2 and 3, alternating the radii
    round by round, --reps rounds after one warm-up: GPU time of the kernel, median, min and max;
  * a full coarse-to-fine alignment (radius 3, then 1, 10 iterations each) of that sweep from a pose 0.3 m / 2 deg
    off: host wall time and iterations, over --reps runs.

    python tools/dense_align_cost.py [--sweeps 55 --leaf 0.1 --reps 15]
"""
from __future__ import annotations

import argparse
import json
import math
import sys
import time

import numpy as np

sys.dont_write_bytecode = True
from dense_cost import dense_ctx, gpu_info, profiled, replay_run, require_cuda, stats  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sweeps", type=int, default=55)
    ap.add_argument("--leaf", type=float, default=0.1)
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()

    require_cuda("dense_align_cost")
    _, _, sweeps, fulls, twists = replay_run(args.sweeps)
    c, voxels = dense_ctx(fulls, args.leaf)

    build = profiled(c, {"build": lambda: c.dense_target_build(None, 2, (0.0, 0.0, 0.0))}, args.reps)["build"]

    # sweep k of the run as the sensor delivered it (sensor frame, not de-skewed), near its mapped pose
    k = args.sweeps // 2
    pts = sweeps[k][0]
    mapped = twists[k]
    it = profiled(c, {f"r{r}": (lambda r=r: c.dense_align_iterate(pts, mapped, r)) for r in (1, 2, 3)}, args.reps)

    rng = np.random.RandomState(3)
    w, u = rng.normal(size=3), rng.normal(size=3)
    init = (mapped + np.concatenate([w / np.linalg.norm(w) * math.radians(2.0), u / np.linalg.norm(u) * 0.3])
            ).astype(np.float32)
    wall, iters = [], []
    for rep in range(args.reps + 1):
        t0 = time.perf_counter()
        a, i1 = c.dense_align(pts, init, 3, 10)
        _, i2 = c.dense_align(pts, a, 1, 10)
        el = time.perf_counter() - t0
        if rep:
            wall.append(1e3 * el)
            iters.append(i1["iterations"] + i2["iterations"])
    c.close()

    print(json.dumps({
        "workload": f"whole-run map of hdl64_1m (BASELINE config 3), {args.sweeps} sweeps replayed at leaf {args.leaf} m;"
                    f" sweep {k} ({pts.shape[0]} points) aligned",
        "voxels": voxels, "target_voxels": build.out, "reps": args.reps,
        "target_build_gpu_ms": stats(build.gpu_ms), "target_build_host_ms": stats(build.host_ms),
        "iteration_gpu_ms": {name: stats(p.gpu_ms) for name, p in it.items()},
        "coarse_to_fine_wall_ms": stats(wall), "coarse_to_fine_iterations": stats(iters),
        "gpu": gpu_info(),
    }))


if __name__ == "__main__":
    main()
