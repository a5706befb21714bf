#!/usr/bin/env python
"""What the visibility pass of the whole-run voxel map costs the streaming pipeline.

Workload: hdl64_1m streaming (tools/dense_cost.py), the whole-run map at --leaf in both arms.  The streaming throughput
is timed with the pass off and on (--h-res / --v-res / --margin), in alternating windows of --steps sweeps on a fresh
pipeline each (after --warmup sweeps), repeated until each arm has --min-seconds of timed windows (at least three);
median, min and max window are reported per arm.  A separate run times the pass's kernels alone: the registered clouds
and poses of the same stream are replayed into a kernel-level context, with CUDA-event profiling (family "dense")
switched on around each dense_observe only.  The hash table's size is read from the library at the end of each arm's
last window and of the replay.  Prints one JSON line.

    python tools/dense_visibility_cost.py [--steps 50 --warmup 5 --leaf 0.1 --min-seconds 0.6]
"""
from __future__ import annotations

import argparse
import json
import sys

import numpy as np

sys.dont_write_bytecode = True
from dense_cost import gpu_info, hdl64_1m, require_cuda, stream_windows  # noqa: E402


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

    require_cuda("dense_visibility_cost")
    from loam_velodyne_b200 import api
    _, _, seed, sweeps = hdl64_1m(args.warmup + args.steps)

    def pipeline(vis):
        p = api.Pipeline()
        p.seed_map(*seed)
        p.mapping.enable_dense_map(args.leaf)
        if vis:
            p.mapping.enable_dense_visibility(args.h_res, args.v_res, args.margin)
        return p

    def probe(p, vis):
        return dict(p.mapping.dense_stats(), table_slots=p.mapping.dense_table_slots())

    rates, probes = stream_windows(args, sweeps, pipeline, (False, True), probe)
    off, on = rates[False], rates[True]
    last = {vis: probes[vis][-1] for vis in (False, True)}

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
