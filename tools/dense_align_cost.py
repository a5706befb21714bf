#!/usr/bin/env python
"""What aligning a sweep against the whole-run voxel map costs.

Workload: the map of tools/dense_normals_cost.py -- BASELINE config 3 (HDL-64E 64 x 2048 sweeps against a 1 M-point
surrounding map), --sweeps sweeps through the pipeline one at a time, their registered clouds replayed into a
kernel-level context with the whole-run map at --leaf.  Reported, with the card's name and power limit read in the same
run:
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
import os
import sys
import time

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
        raise SystemExit("dense_align_cost: no CUDA device (nothing here runs on the CPU)")
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

    build_gpu, build_host = [], []
    for rep in range(args.reps + 1):
        c.profile(True)
        t0 = time.perf_counter()
        n_target = c.dense_target_build(None, 2, (0.0, 0.0, 0.0))
        el = time.perf_counter() - t0
        if rep:
            build_gpu.append(c.profile_get()["dense"][0])
            build_host.append(1e3 * el)

    # sweep k of the run as the sensor delivered it (sensor frame, not de-skewed), near its mapped pose
    k = args.sweeps // 2
    pts, _ = synth.make_sweep(scene, lidar, k, yaw_rate=math.radians(5.0))
    mapped = twists[k]
    it_gpu = {r: [] for r in (1, 2, 3)}
    for rep in range(args.reps + 1):
        for r in (1, 2, 3):
            c.profile(True)
            c.dense_align_iterate(pts, mapped, r)
            if rep:
                it_gpu[r].append(c.profile_get()["dense"][0])

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
        "voxels": voxels, "target_voxels": n_target, "reps": args.reps,
        "target_build_gpu_ms": stats(build_gpu), "target_build_host_ms": stats(build_host),
        "iteration_gpu_ms": {f"r{r}": stats(v) for r, v in it_gpu.items()},
        "coarse_to_fine_wall_ms": stats(wall), "coarse_to_fine_iterations": stats(iters),
        "gpu": gpu_info(),
    }))


if __name__ == "__main__":
    main()
