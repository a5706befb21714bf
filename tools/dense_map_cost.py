#!/usr/bin/env python
"""What the whole-run voxel map costs the streaming pipeline.

Workload: hdl64_1m streaming (tools/dense_cost.py), the map at --leaf.  The streaming throughput is timed with the map
off and on, in alternating windows of --steps sweeps on a fresh pipeline each (after --warmup sweeps), repeated until
each arm has --min-seconds of timed windows (at least three); median, min and max window are reported per arm.  A
separate run times the insertion kernels alone: the registered clouds of the same stream are replayed into a
kernel-level context with CUDA-event profiling (family "dense"), and the host time the mapping thread spends per sweep
(its stage's busy time while streaming, its end-of-sweep call one sweep at a time) is reported with the map off and on.
Prints one JSON line.

    python tools/dense_map_cost.py [--steps 50 --warmup 5 --leaf 0.1 --min-seconds 0.6]
"""
from __future__ import annotations

import argparse
import json
import sys

import numpy as np

sys.dont_write_bytecode = True
from dense_cost import dense_ctx, gpu_info, hdl64_1m, require_cuda, stream_windows  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--leaf", type=float, default=0.1)
    ap.add_argument("--min-seconds", type=float, default=0.6)
    ap.add_argument("--max-windows", type=int, default=40)
    args = ap.parse_args()

    require_cuda("dense_map_cost")
    import torch
    from loam_velodyne_b200 import api
    _, _, seed, sweeps = hdl64_1m(args.warmup + args.steps)

    def pipeline(dense):
        p = api.Pipeline()
        p.seed_map(*seed)
        if dense:
            p.mapping.enable_dense_map(args.leaf)
        return p

    def probe(p, dense):
        busy = p.stage_seconds()["busy"] / args.steps  # host seconds per sweep inside each stage's work
        stats = p.mapping.dense_stats() if dense else None
        return busy, stats, torch.cuda.mem_get_info()[0]

    rates, probes = stream_windows(args, sweeps, pipeline, (False, True), probe)
    off, on = rates[False], rates[True]
    busy = {d: round(1e3 * float(np.median([b[2] for b, _, _ in probes[d]])), 4) for d in (False, True)}
    last = probes[True][-1][1]

    # host side: the mapping thread's end-of-sweep call (transform + insertion issue + hand-off to the helper thread)
    # per sweep, one sweep at a time, map off and on; the registered clouds of the stream for the replay below
    end_ms = {}
    fulls = []
    for dense in (False, True):
        seq = pipeline(dense)
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
    c, _ = dense_ctx(fulls[:args.warmup], args.leaf)
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
        "mapping_stage_busy_ms_per_sweep_median": {"off": busy[False], "on": busy[True]},
        "end_sweep_call_ms_median": {"off": round(end_ms[False], 4), "on": round(end_ms[True], 4)},
        "dense_gpu_ms_per_sweep": round(ms / max(len(fulls) - args.warmup, 1), 4),
        "dense_launches_per_sweep": round(launches / max(len(fulls) - args.warmup, 1), 2),
        "points_per_sweep": int(np.mean([f.shape[0] for f in fulls])),
        "voxels_after_run": voxels, "skipped": last["skipped"], "dropped": last["dropped"],
        "replay_voxels": replay["voxels"],
        "table_bytes_at_least": slots * 48,
        "device_bytes_map_on_minus_off": int(probes[False][-1][2] - probes[True][-1][2]),
        "gpu": gpu_info(),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
