#!/usr/bin/env python
"""What ray casting the whole-run voxel map costs.

Workload: the replayed hdl64_1m map (tools/dense_cost.py), --sweeps sweeps at --leaf, and the target built from it
(radius 2).  Reported, with the card's name and power limit read in the same run:
  * the first cast after the build (64 x 2048 grid, max_range 100 m): GPU time including the ray index build
    (CUDA-event profiling, family "dense"), over --reps builds;
  * later casts of a 64 x 2048 lidar_rays grid at max_range 50, 100 and 200 m, and of a 131 k-point sweep's own
    points at 100 m, alternating the four round by round, --reps rounds after one warm-up: GPU time of the kernel,
    median, min and max;
  * the ray index's device bytes.

    python tools/dense_raycast_cost.py [--sweeps 55 --leaf 0.1 --reps 15]
"""
from __future__ import annotations

import argparse
import json
import sys

import numpy as np

sys.dont_write_bytecode = True
from dense_cost import dense_ctx, gpu_info, profiled, replay_run, require_cuda, stats  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sweeps", type=int, default=55)
    ap.add_argument("--leaf", type=float, default=0.1)
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()

    require_cuda("dense_raycast_cost")
    from loam_velodyne_b200 import api
    _, lidar, sweeps, fulls, twists = replay_run(args.sweeps)
    c, voxels = dense_ctx(fulls, args.leaf)

    k = args.sweeps // 2
    pose = twists[k]
    grid = api.lidar_rays(np.linspace(lidar.lower_deg, lidar.upper_deg, lidar.n_rings), 2048)
    pts = sweeps[k][0]

    first = []
    for rep in range(args.reps + 1):
        n_target = c.dense_target_build(None, 2, (0.0, 0.0, 0.0))
        c.profile(True)
        c.dense_raycast(grid, pose, 0.0, 100.0)
        if rep:
            first.append(c.profile_get()["dense"][0])
    index_bytes = c.dense_ray_index_bytes()

    cases = {"grid_50m": (grid, 50.0), "grid_100m": (grid, 100.0), "grid_200m": (grid, 200.0),
             "sweep_100m": (pts, 100.0)}
    later = profiled(c, {name: (lambda rays=rays, mx=mx: c.dense_raycast(rays, pose, 0.0, mx))
                         for name, (rays, mx) in cases.items()}, args.reps)
    c.close()

    print(json.dumps({
        "workload": f"whole-run map of hdl64_1m (BASELINE config 3), {args.sweeps} sweeps replayed at leaf {args.leaf} m;"
                    f" cast from sweep {k}'s mapped pose: a 64 x 2048 grid, sweep {k}'s own {pts.shape[0]} points",
        "voxels": voxels, "target_voxels": n_target, "reps": args.reps, "ray_index_bytes": index_bytes,
        "first_cast_with_index_gpu_ms": stats(first),
        "cast_gpu_ms": {name: stats(p.gpu_ms) for name, p in later.items()},
        "hit_fraction": {name: round(float(np.isfinite(p.out[0]).mean()), 4) for name, p in later.items()},
        "gpu": gpu_info(),
    }))


if __name__ == "__main__":
    main()
