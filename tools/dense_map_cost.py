#!/usr/bin/env python
"""What the whole-run voxel map costs the streaming pipeline.

Workload: BASELINE config 3 (HDL-64E 64 x 2048 sweeps against a 1 M-point surrounding map), the map at --leaf.  The
streaming throughput is timed with the map off and on, in alternating windows of --steps sweeps on a fresh pipeline
each (after --warmup sweeps), repeated until each arm has --min-seconds of timed windows (at least three); median, min
and max window are reported per arm.  A separate run times the insertion kernels alone: the registered clouds of the
same stream are replayed into a kernel-level context with CUDA-event profiling (family "dense"), and the host time the
mapping thread spends per sweep (its stage's busy time while streaming, its end-of-sweep call one sweep at a time) is
reported with the map off and on.  Prints one JSON line.

    python tools/dense_map_cost.py [--steps 50 --warmup 5 --leaf 0.1 --min-seconds 0.6]
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
    ap.add_argument("--min-seconds", type=float, default=0.6)
    ap.add_argument("--max-windows", type=int, default=40)
    args = ap.parse_args()

    import torch
    from loam_velodyne_b200 import api, synth
    if not torch.cuda.is_available():
        raise SystemExit("dense_map_cost: no CUDA device (nothing here runs on the CPU)")
    scene = synth.make_scene()
    lidar = synth.Lidar.hdl64()
    corner, surf = synth.make_map(scene, 1_000_000)
    n = args.warmup + args.steps
    sweeps = [synth.make_sweep(scene, lidar, i, yaw_rate=math.radians(5.0)) for i in range(n)]
    d_sweeps = [torch.from_numpy(p).to("cuda:0") for p, _ in sweeps]
    torch.cuda.synchronize()

    def window(dense):
        p = api.Pipeline()
        p.seed_map(corner, surf)
        if dense:
            p.mapping.enable_dense_map(args.leaf)

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
        p.stage_seconds(reset=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run(args.warmup, n)  # ends with every stage (and the map insertion) finished on the GPU
        torch.cuda.synchronize()
        el = time.perf_counter() - t0
        busy = p.stage_seconds()["busy"] / args.steps  # host seconds per sweep inside each stage's work
        stats = p.mapping.dense_stats() if dense else None
        free = torch.cuda.mem_get_info()[0]
        del p
        return el, stats, free, busy

    windows = {False: [], True: []}
    busy_of = {False: [], True: []}
    last = {}
    free_of = {}
    while True:
        for dense in (False, True):
            el, stats, free, busy = window(dense)
            windows[dense].append(el)
            busy_of[dense].append(busy)
            free_of[dense] = free
            if dense:
                last = stats
        done = [sum(windows[d]) >= args.min_seconds and len(windows[d]) >= 3 for d in (False, True)]
        if all(done) or len(windows[True]) >= args.max_windows:
            break

    def arm(els):
        s = sorted(els)
        sps = [args.steps / e for e in s]
        return {"sweeps_per_s_median": round(args.steps / s[len(s) // 2], 1), "sweeps_per_s_min": round(min(sps), 1),
                "sweeps_per_s_max": round(max(sps), 1), "windows": len(s),
                "window_ms_min_median_max": [round(1e3 * s[0], 2), round(1e3 * s[len(s) // 2], 2), round(1e3 * s[-1], 2)]}

    off, on = arm(windows[False]), arm(windows[True])

    # host side: the mapping thread's end-of-sweep call (transform + insertion issue + hand-off to the helper thread)
    # per sweep, one sweep at a time, map off and on; the registered clouds of the stream for the replay below
    end_ms = {}
    fulls = []
    for dense in (False, True):
        seq = api.Pipeline()
        seq.seed_map(corner, surf)
        if dense:
            seq.mapping.enable_dense_map(args.leaf)
        ph = []
        for i, (pts, rs) in enumerate(sweeps):
            seq.sweep(pts, rs)
            if i >= args.warmup:
                ph.append(seq.mapping.last_phase_ms()["end_sweep"])
            if not dense:
                fulls.append(seq.mapping.cloud("full"))
        seq.sync()
        del seq
        end_ms[dense] = float(np.median(ph))

    # the insertion kernels alone: the registered clouds of the same stream, replayed with CUDA-event profiling
    c = api.Ctx(0)
    c.dense_enable(args.leaf)
    for f in fulls[:args.warmup]:
        c.cloud_upload(api.C_MAP_FULL, f)
        c.dense_insert(api.C_MAP_FULL)
    c.profile(True)
    for f in fulls[args.warmup:]:
        c.cloud_upload(api.C_MAP_FULL, f)
        c.dense_insert(api.C_MAP_FULL)
    ms, launches = c.profile_get()["dense"]
    replay = c.dense_stats()
    c.close()

    voxels = last["voxels"]
    slots = 1024
    while slots < 2 * voxels:
        slots *= 2
    out = {
        "workload": "hdl64_1m streaming (BASELINE config 3), inputs in HBM",
        "leaf_m": args.leaf, "steps": args.steps, "warmup": args.warmup,
        "map_off": off, "map_on": on,
        "throughput_change_pct": round(100.0 * (on["sweeps_per_s_median"] / off["sweeps_per_s_median"] - 1.0), 2),
        "mapping_stage_busy_ms_per_sweep_median": {"off": round(1e3 * float(np.median([b[2] for b in busy_of[False]])), 4),
                                                   "on": round(1e3 * float(np.median([b[2] for b in busy_of[True]])), 4)},
        "end_sweep_call_ms_median": {"off": round(end_ms[False], 4), "on": round(end_ms[True], 4)},
        "dense_gpu_ms_per_sweep": round(ms / max(len(fulls) - args.warmup, 1), 4),
        "dense_launches_per_sweep": round(launches / max(len(fulls) - args.warmup, 1), 2),
        "points_per_sweep": int(np.mean([f.shape[0] for f in fulls])),
        "voxels_after_run": voxels, "skipped": last["skipped"], "dropped": last["dropped"],
        "replay_voxels": replay["voxels"],
        "table_bytes_at_least": slots * 48,
        "device_bytes_map_on_minus_off": int(free_of[False] - free_of[True]),
        "gpu": gpu_info(),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
