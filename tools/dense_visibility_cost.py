#!/usr/bin/env python
"""What the visibility pass of the whole-run voxel map costs the streaming pipeline.

Workload: BASELINE config 3 (HDL-64E 64 x 2048 sweeps against a 1 M-point surrounding map), the whole-run map at
--leaf in both arms.  The streaming throughput is timed with the pass off and on (--h-res / --v-res / --margin), in
alternating windows of --steps sweeps on a fresh pipeline each (after --warmup sweeps), repeated until each arm has
--min-seconds of timed windows (at least three); median, min and max window are reported per arm.  A separate run
times the pass's kernels alone: the registered clouds and poses of the same stream are replayed into a kernel-level
context, with CUDA-event profiling (family "dense") switched on around each dense_observe only.  The hash table's size
is read from the library at the end of each arm's last window and of the replay.  Prints one JSON line.

    python tools/dense_visibility_cost.py [--steps 50 --warmup 5 --leaf 0.1 --min-seconds 0.6]
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
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--leaf", type=float, default=0.1)
    ap.add_argument("--h-res", type=float, default=1.0)
    ap.add_argument("--v-res", type=float, default=2.0)
    ap.add_argument("--margin", type=float, default=1.0)
    ap.add_argument("--min-seconds", type=float, default=0.6)
    ap.add_argument("--max-windows", type=int, default=40)
    args = ap.parse_args()

    import torch
    from loam_velodyne_b200 import api, synth
    if not torch.cuda.is_available():
        raise SystemExit("dense_visibility_cost: no CUDA device (nothing here runs on the CPU)")
    scene = synth.make_scene()
    lidar = synth.Lidar.hdl64()
    corner, surf = synth.make_map(scene, 1_000_000)
    n = args.warmup + args.steps
    sweeps = [synth.make_sweep(scene, lidar, i, yaw_rate=math.radians(5.0)) for i in range(n)]
    d_sweeps = [torch.from_numpy(p).to("cuda:0") for p, _ in sweeps]
    torch.cuda.synchronize()

    def pipeline(vis):
        p = api.Pipeline()
        p.seed_map(corner, surf)
        p.mapping.enable_dense_map(args.leaf)
        if vis:
            p.mapping.enable_dense_visibility(args.h_res, args.v_res, args.margin)
        return p

    def window(vis):
        p = pipeline(vis)

        def run(lo, hi):
            got = 0
            for i in range(lo, hi):
                p.submit(ring_sizes=sweeps[i][1], device_ptr=d_sweeps[i].data_ptr())
                if p.collect(wait=False) is not None:
                    got += 1
            while got < hi - lo:
                p.collect(wait=True)
                got += 1
            p.sync()

        run(0, args.warmup)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run(args.warmup, n)  # ends with every stage (and the map's pass and insertion) finished on the GPU
        torch.cuda.synchronize()
        el = time.perf_counter() - t0
        stats = dict(p.mapping.dense_stats(), table_slots=p.mapping.dense_table_slots())
        del p
        return el, stats

    windows = {False: [], True: []}
    last = {}
    while True:
        for vis in (False, True):
            el, stats = window(vis)
            windows[vis].append(el)
            last[vis] = stats
        done = [sum(windows[v]) >= args.min_seconds and len(windows[v]) >= 3 for v in (False, True)]
        if all(done) or len(windows[True]) >= args.max_windows:
            break

    def arm(els):
        s = sorted(els)
        sps = [args.steps / e for e in s]
        return {"sweeps_per_s_median": round(args.steps / s[len(s) // 2], 1), "sweeps_per_s_min": round(min(sps), 1),
                "sweeps_per_s_max": round(max(sps), 1), "windows": len(s),
                "window_ms_min_median_max": [round(1e3 * s[0], 2), round(1e3 * s[len(s) // 2], 2), round(1e3 * s[-1], 2)]}

    off, on = arm(windows[False]), arm(windows[True])

    # the registered clouds and optimised poses of the stream, one sweep at a time
    seq = pipeline(True)
    fulls, poses = [], []
    for pts, rs in sweeps:
        seq.sweep(pts, rs)
        fulls.append(seq.mapping.cloud("full"))
        poses.append(seq.mapping.twist("tobe"))
    removed = seq.mapping.dense_stats()["voxels"] - seq.mapping.dense_map(1.0)[0].shape[0]
    seq.sync()
    del seq

    # the pass's kernels alone (memset + range image + table scan), replayed with CUDA-event profiling around each pass
    c = api.Ctx(0)
    c.dense_enable(args.leaf)
    c.dense_visibility(args.h_res, args.v_res, args.margin)
    c.profile(False)
    ms_list = []
    for i, (f, pose) in enumerate(zip(fulls, poses)):
        c.cloud_upload(api.C_MAP_FULL, f)
        if i >= args.warmup:
            c.profile(True)
        c.dense_observe(api.C_MAP_FULL, pose)
        if i >= args.warmup:
            ms_list.append(c.profile_get()["dense"])
            c.L.loam_b200_profile_enable(c.h, 0)
        c.dense_insert(api.C_MAP_FULL)
    replay = dict(c.dense_stats(), table_slots=c.dense_table_slots())
    c.close()
    ms = [m for m, _ in ms_list]

    out = {
        "workload": "hdl64_1m streaming (BASELINE config 3), inputs in HBM, whole-run map on in both arms",
        "leaf_m": args.leaf, "h_res_deg": args.h_res, "v_res_deg": args.v_res, "margin_m": args.margin,
        "steps": args.steps, "warmup": args.warmup,
        "pass_off": off, "pass_on": on,
        "throughput_change_pct": round(100.0 * (on["sweeps_per_s_median"] / off["sweeps_per_s_median"] - 1.0), 2),
        "visibility_gpu_ms_per_sweep_median": round(float(np.median(ms)), 4),
        "visibility_gpu_ms_per_sweep_last": round(ms[-1], 4),
        "visibility_launches_per_sweep": round(ms_list[-1][1], 2),
        "points_per_sweep": int(np.mean([f.shape[0] for f in fulls])),
        "voxels_after_run": last[True]["voxels"], "replay_voxels": replay["voxels"],
        "table_slots_read_from_library": {"pass_off": last[False]["table_slots"], "pass_on": last[True]["table_slots"],
                                          "replay": replay["table_slots"]},
        "table_bytes_pass_on": last[True]["table_slots"] * 48,
        "voxels_removed_at_ratio_1": int(removed),
        "gpu": gpu_info(),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
