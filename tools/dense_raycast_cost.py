#!/usr/bin/env python
"""What ray casting the whole-run voxel map costs.

Workload: the map of tools/dense_align_cost.py -- BASELINE config 3 (HDL-64E 64 x 2048 sweeps against a 1 M-point
surrounding map), --sweeps sweeps through the pipeline, their registered clouds replayed into a kernel-level context
with the whole-run map at --leaf, and the target built from it (radius 2).  Reported, with the card's name and power
limit read in the same run:
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
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True


def gpu_info():
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(0)
        name = pynvml.nvmlDeviceGetName(h)
        return {"name": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": round(pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0, 1)}
    except Exception:
        import subprocess
        try:
            out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                 stdout=subprocess.PIPE, text=True, check=True).stdout.strip().splitlines()[0]
            name, limit = (s.strip() for s in out.split(","))
            return {"name": name, "power_limit": limit}
        except Exception:
            import torch
            return {"name": torch.cuda.get_device_name(0), "power_limit_w": None}


def stats(v):
    return {"median": round(float(np.median(v)), 4), "min": round(float(np.min(v)), 4),
            "max": round(float(np.max(v)), 4)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sweeps", type=int, default=55)
    ap.add_argument("--leaf", type=float, default=0.1)
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()

    import torch
    from loam_velodyne_b200 import api, synth
    if not torch.cuda.is_available():
        raise SystemExit("dense_raycast_cost: no CUDA device (nothing here runs on the CPU)")
    scene = synth.make_scene()
    lidar = synth.Lidar.hdl64()
    corner, surf = synth.make_map(scene, 1_000_000)
    seq = api.Pipeline()
    seq.seed_map(corner, surf)
    fulls, twists = [], []
    for i in range(args.sweeps):
        seq.sweep(*synth.make_sweep(scene, lidar, i, yaw_rate=math.radians(5.0)))
        fulls.append(seq.mapping.cloud("full"))
        twists.append(seq.mapping.twist("aft"))
    seq.sync()
    del seq

    c = api.Ctx(0)
    c.dense_enable(args.leaf)
    for f in fulls:
        c.cloud_upload(api.C_MAP_FULL, f)
        c.dense_insert(api.C_MAP_FULL)
    voxels = c.dense_stats()["voxels"]

    k = args.sweeps // 2
    pose = twists[k]
    grid = api.lidar_rays(np.linspace(lidar.lower_deg, lidar.upper_deg, lidar.n_rings), 2048)
    pts, _ = synth.make_sweep(scene, lidar, k, yaw_rate=math.radians(5.0))

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
    later = {name: [] for name in cases}
    hits = {}
    for rep in range(args.reps + 1):
        for name, (rays, mx) in cases.items():
            c.profile(True)
            r, _ = c.dense_raycast(rays, pose, 0.0, mx)
            if rep:
                later[name].append(c.profile_get()["dense"][0])
            hits[name] = round(float(np.isfinite(r).mean()), 4)
    c.close()

    print(json.dumps({
        "workload": f"whole-run map of hdl64_1m (BASELINE config 3), {args.sweeps} sweeps replayed at leaf {args.leaf} m;"
                    f" cast from sweep {k}'s mapped pose: a 64 x 2048 grid, sweep {k}'s own {pts.shape[0]} points",
        "voxels": voxels, "target_voxels": n_target, "reps": args.reps, "ray_index_bytes": index_bytes,
        "first_cast_with_index_gpu_ms": stats(first),
        "cast_gpu_ms": {name: stats(v) for name, v in later.items()}, "hit_fraction": hits,
        "gpu": gpu_info(),
    }))


if __name__ == "__main__":
    main()
