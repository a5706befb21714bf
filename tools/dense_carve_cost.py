#!/usr/bin/env python
"""What carve mode of the whole-run voxel map's visibility pass costs, beside the range-image mode.

Workload: hdl64_1m streaming (tools/dense_cost.py), the whole-run map at --leaf in every arm.  The streaming
throughput is timed for the map only, the range-image mode (1 deg x 2 deg, 1 m) and carve mode (--margin,
--max-range), in alternating windows of --steps sweeps on a fresh pipeline each (after --warmup sweeps), repeated until
each arm has --min-seconds of timed windows (at least three).  Kernel times come from a replay of the stream's
registered clouds and poses into a kernel-level context, with CUDA-event profiling (family "dense") switched on around
one call at a time:
  * the carve pass per sweep at max_range 50 m and 100 m, and the insertion with carve mode off and on (the difference
    is the index's incremental update);
  * both modes' passes at two map sizes: the run's own map, then the same sweeps replayed --replicas more times,
    shifted by 500 m each along x, so the table is several times larger while the observed sweeps stay the same.
Prints one JSON line.

    python tools/dense_carve_cost.py [--steps 50 --warmup 5 --leaf 0.1 --min-seconds 0.6]
"""
from __future__ import annotations

import argparse
import json
import sys

import numpy as np

sys.dont_write_bytecode = True
from dense_cost import gpu_info, hdl64_1m, require_cuda, stats, stream_windows  # noqa: E402

H_RES, V_RES, VIS_MARGIN = 1.0, 2.0, 1.0


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--leaf", type=float, default=0.1)
    ap.add_argument("--margin", type=float, default=2.0)
    ap.add_argument("--max-range", type=float, default=100.0)
    ap.add_argument("--replicas", type=int, default=4)
    ap.add_argument("--min-seconds", type=float, default=0.6)
    ap.add_argument("--max-windows", type=int, default=20)
    args = ap.parse_args()

    require_cuda("dense_carve_cost")
    from loam_velodyne_b200 import api
    _, _, seed, sweeps = hdl64_1m(args.warmup + args.steps)
    arms = ("map_only", "range_image", "carve")

    def pipeline(arm):
        p = api.Pipeline()
        p.seed_map(*seed)
        p.mapping.enable_dense_map(args.leaf)
        if arm == "range_image":
            p.mapping.enable_dense_visibility(H_RES, V_RES, VIS_MARGIN)
        elif arm == "carve":
            p.mapping.enable_dense_carving(args.margin, args.max_range)
        return p

    rates, _ = stream_windows(args, sweeps, pipeline, arms)
    streaming = {a: {k: v for k, v in r.items() if k != "window_ms_min_median_max"} for a, r in rates.items()}

    # the registered clouds and optimised poses of the stream (the pass never changes them)
    seq = pipeline("map_only")
    fulls, poses = [], []
    for pts, rs in sweeps:
        seq.sweep(pts, rs)
        fulls.append(seq.mapping.cloud("full"))
        poses.append(seq.mapping.twist("tobe"))
    seq.sync()
    del seq

    def timed(c, fn):
        c.profile(True)
        fn()
        ms, launches = c.profile_get()["dense"]
        c.L.loam_b200_profile_enable(c.h, 0)
        return ms, launches

    def replay(max_range):
        """carve pass and insertion per sweep (carve on), and the insertion alone (carve off)."""
        out = {"observe": [], "insert_on": [], "insert_off": []}
        for carve in (False, True):
            c = api.Ctx(0)
            c.dense_enable(args.leaf)
            if carve:
                c.dense_carving(args.margin, max_range)
            for i, (f, pose) in enumerate(zip(fulls, poses)):
                c.cloud_upload(api.C_MAP_FULL, f)
                if carve:
                    ms = timed(c, lambda: c.dense_observe(api.C_MAP_FULL, pose))
                    if i >= args.warmup:
                        out["observe"].append(ms)
                ms = timed(c, lambda: c.dense_insert(api.C_MAP_FULL))
                if i >= args.warmup:
                    out["insert_on" if carve else "insert_off"].append(ms)
            if carve:
                out["voxels"] = c.dense_stats()["voxels"]
                out["bricks"] = int(c.dense_carve_index()[0].size)
            c.close()
        return out

    per_range = {mr: replay(mr) for mr in (50.0, args.max_range)}
    main_r = per_range[args.max_range]

    # scaling: both passes over the last --steps sweeps at the run's map size, then after --replicas shifted replays
    c = api.Ctx(0)
    c.dense_enable(args.leaf)

    def insert_all(shift):
        for f in fulls:
            g = f.copy()
            g[:, 0] += np.float32(shift)
            c.cloud_upload(api.C_MAP_FULL, g)
            c.dense_insert(api.C_MAP_FULL)

    def both_passes():
        res = {}
        c.dense_visibility(H_RES, V_RES, VIS_MARGIN)
        ri = []
        for f, pose in zip(fulls[args.warmup:], poses[args.warmup:]):
            c.cloud_upload(api.C_MAP_FULL, f)
            ri.append(timed(c, lambda: c.dense_observe(api.C_MAP_FULL, pose))[0])
        c.dense_visibility(0.0, 0.0, 0.0)
        c.dense_carving(args.margin, args.max_range)
        cv = []
        for f, pose in zip(fulls[args.warmup:], poses[args.warmup:]):
            c.cloud_upload(api.C_MAP_FULL, f)
            cv.append(timed(c, lambda: c.dense_observe(api.C_MAP_FULL, pose))[0])
        c.dense_carving(0.0, 0.0)
        res["range_image_gpu_ms_median"] = stats(ri)["median"]
        res["carve_gpu_ms_median"] = stats(cv)["median"]
        res["voxels"] = c.dense_stats()["voxels"]
        res["table_slots"] = c.dense_table_slots()
        return res

    insert_all(0.0)
    scaling = [both_passes()]
    for k in range(1, args.replicas + 1):
        insert_all(500.0 * k)
    scaling.append(both_passes())
    c.close()
    insert_ms = {k: stats([m for m, _ in main_r[f"insert_{k}"]])["median"] for k in ("off", "on")}

    out = {
        "workload": "hdl64_1m streaming (BASELINE config 3), inputs in HBM, whole-run map on in every arm",
        "leaf_m": args.leaf, "carve_margin_m": args.margin, "carve_max_range_m": args.max_range,
        "range_image": {"h_res_deg": H_RES, "v_res_deg": V_RES, "margin_m": VIS_MARGIN},
        "steps": args.steps, "warmup": args.warmup,
        "streaming": streaming,
        "carve_change_vs_map_only_pct": round(100.0 * (streaming["carve"]["sweeps_per_s_median"] /
                                                       streaming["map_only"]["sweeps_per_s_median"] - 1.0), 2),
        "range_image_change_vs_map_only_pct": round(100.0 * (streaming["range_image"]["sweeps_per_s_median"] /
                                                             streaming["map_only"]["sweeps_per_s_median"] - 1.0), 2),
        "carve_gpu_ms_per_sweep_median": {f"{mr:g}m": stats([m for m, _ in r["observe"]])["median"]
                                          for mr, r in per_range.items()},
        "carve_launches_per_sweep": main_r["observe"][-1][1],
        "insert_gpu_ms_median": {"carve_off": insert_ms["off"], "carve_on": insert_ms["on"]},
        "index_update_gpu_ms_per_sweep": round(insert_ms["on"] - insert_ms["off"], 4),
        "insert_launches": {"carve_off": main_r["insert_off"][-1][1], "carve_on": main_r["insert_on"][-1][1]},
        "points_per_sweep": int(np.mean([f.shape[0] for f in fulls])),
        "voxels_after_run": main_r["voxels"], "index_bricks": main_r["bricks"],
        "scaling": scaling,
        "gpu": gpu_info(),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
