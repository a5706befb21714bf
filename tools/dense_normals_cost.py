#!/usr/bin/env python
"""What the normals of the whole-run voxel map cost at export.

Workload: the map of tools/dense_map_cost.py -- BASELINE config 3 (HDL-64E 64 x 2048 sweeps against a 1 M-point
surrounding map), --sweeps sweeps through the pipeline one at a time, their registered clouds replayed into a
kernel-level context with the whole-run map at --leaf.  Then, alternating and repeated --reps times after one warm-up
round, the filtered export (dense_export at ratio +inf) and the export with normals at radius 1, 2 and 3: the host
time of each synchronous call (perf_counter around it) and the GPU time of its kernels (CUDA-event profiling, family
"dense", reset before each call).  Prints one JSON line with medians, min and max, the voxel count, and the card's
name and power limit read in the same run.

    python tools/dense_normals_cost.py [--sweeps 55 --leaf 0.1 --reps 15]
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


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sweeps", type=int, default=55)
    ap.add_argument("--leaf", type=float, default=0.1)
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()

    import torch
    from loam_velodyne_b200 import api, synth
    if not torch.cuda.is_available():
        raise SystemExit("dense_normals_cost: no CUDA device (nothing here runs on the CPU)")
    scene = synth.make_scene()
    lidar = synth.Lidar.hdl64()
    corner, surf = synth.make_map(scene, 1_000_000)
    seq = api.Pipeline()
    seq.seed_map(corner, surf)
    fulls = []
    for i in range(args.sweeps):
        seq.sweep(*synth.make_sweep(scene, lidar, i, yaw_rate=math.radians(5.0)))
        fulls.append(seq.mapping.cloud("full"))
    seq.sync()
    del seq

    c = api.Ctx(0)
    c.dense_enable(args.leaf)
    for f in fulls:
        c.cloud_upload(api.C_MAP_FULL, f)
        c.dense_insert(api.C_MAP_FULL)
    voxels = c.dense_stats()["voxels"]

    arms = {"filtered": lambda: c.dense_export(math.inf)}
    for r in (1, 2, 3):
        arms[f"normals_r{r}"] = (lambda r=r: c.dense_export_normals(math.inf, r, (0.0, 0.0, 0.0)))
    host = {k: [] for k in arms}
    gpu = {k: [] for k in arms}
    launches = {}
    undefined = {}
    for rep in range(args.reps + 1):
        for name, fn in arms.items():
            c.profile(True)  # on + reset
            t0 = time.perf_counter()
            out = fn()
            el = time.perf_counter() - t0
            ms, n = c.profile_get()["dense"]
            if rep == 0:
                continue  # warm-up round
            host[name].append(1e3 * el)
            gpu[name].append(ms)
            launches[name] = n
            if name != "filtered":
                undefined[name] = int(np.isnan(out[2][:, 0]).sum())
    c.close()

    def stats(v):
        return {"median": round(float(np.median(v)), 4), "min": round(float(np.min(v)), 4),
                "max": round(float(np.max(v)), 4)}

    out = {
        "workload": f"whole-run map of hdl64_1m (BASELINE config 3), {args.sweeps} sweeps replayed at leaf {args.leaf} m",
        "voxels": voxels, "reps": args.reps,
        "host_ms_per_call": {k: stats(v) for k, v in host.items()},
        "gpu_ms_per_call": {k: stats(v) for k, v in gpu.items()},
        "normals_gpu_ms_over_filtered_median": {k: round(float(np.median(gpu[k]) - np.median(gpu["filtered"])), 4)
                                                for k in arms if k != "filtered"},
        "launches_per_call": launches,
        "undefined_normals": undefined,
        "gpu": gpu_info(),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
