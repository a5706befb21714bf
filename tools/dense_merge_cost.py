#!/usr/bin/env python
"""What snapshots and merging of the whole-run voxel map cost.

Workload: the replayed hdl64_1m map (tools/dense_cost.py), --sweeps sweeps at --leaf (55 at 0.1 m: the config-3 map).
Reported, with the card's name and power limit read in the same run, each over --reps rounds after one warm-up:
  * the snapshot: GPU time (CUDA-event profiling, family "dense") and host wall time of the whole call (readback of
    the 40 bytes per voxel and the evidence unpacking included);
  * resume: the snapshot merged with no pose into a context whose map was just cleared (the table keeps its size, so
    no growth is timed): GPU time and host wall time (the upload included);
  * the map merged into itself under a pose of 1 m and 5 deg of yaw: the same context cleared and resumed first (not
    timed), then the merge timed -- about half the entries land in stored voxels, half in new ones.

    python tools/dense_merge_cost.py [--sweeps 55 --leaf 0.1 --reps 10]
"""
from __future__ import annotations

import argparse
import json
import math
import sys
import time

sys.dont_write_bytecode = True
from dense_cost import dense_ctx, gpu_info, profiled, replay_run, require_cuda, stats  # noqa: E402

POSE = (0.0, math.radians(5.0), 0.0, 0.6, 0.0, 0.8)  # 5 deg of yaw, 1 m on the ground plane


def timed_merges(d, snap, reps, twist):
    """reps + 1 rounds (the first a warm-up) of: clear, resume (untimed unless twist is None), merge under twist ->
    (GPU ms, host ms, launches of the timed merge, voxels after it)."""
    gpu, host, launches, voxels = [], [], 0, 0
    for rep in range(reps + 1):
        d.dense_clear()
        if twist is not None:
            d.dense_merge(snap)
            d.dense_stats()
        d.profile(True)
        t0 = time.perf_counter()
        d.dense_merge(snap, twist)
        voxels = d.dense_stats()["voxels"]  # synchronises: the merge has finished
        el = time.perf_counter() - t0
        ms, launches = d.profile_get()["dense"]
        if rep:
            gpu.append(ms)
            host.append(1e3 * el)
    return gpu, host, launches, voxels


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sweeps", type=int, default=55)
    ap.add_argument("--leaf", type=float, default=0.1)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()

    require_cuda("dense_merge_cost")
    from loam_velodyne_b200 import api
    _, _, _, fulls, _ = replay_run(args.sweeps)
    c, voxels = dense_ctx(fulls, args.leaf)
    snap = profiled(c, {"snapshot": c.dense_snapshot}, args.reps)["snapshot"]
    s = snap.out
    assert s["keys"].size == voxels
    c.close()

    d = api.Ctx(0)
    d.dense_enable(args.leaf)
    out = {}
    for name, twist in (("resume", None), ("self_under_pose", POSE)):
        gpu, host, launches, after = timed_merges(d, s, args.reps, twist)
        out[name] = {"gpu_ms": stats(gpu), "host_ms": stats(host), "launches": launches, "voxels_after": after,
                     "entries_per_s": round(voxels / (float(sorted(gpu)[len(gpu) // 2]) * 1e-3), 1)}
    d.close()

    print(json.dumps({
        "workload": f"whole-run map of hdl64_1m (BASELINE config 3), {args.sweeps} sweeps replayed at leaf {args.leaf} m",
        "voxels": voxels, "reps": args.reps, "pose": [round(float(x), 6) for x in POSE],
        "snapshot": {"gpu_ms": stats(snap.gpu_ms), "host_ms": stats(snap.host_ms), "launches": snap.launches,
                     "bytes_out": int(voxels * 40)},
        "merge": out, "gpu": gpu_info(),
    }))


if __name__ == "__main__":
    main()
