#!/usr/bin/env python
"""What place recognition and global relocalisation in the whole-run voxel map cost.

Workloads, with the card's name and power limit read in the same run:
  * the replayed hdl64_1m map of tools/dense_cost.py, --sweeps sweeps at --leaf, target radius 2;
  * the route map of tests/test_dense_place.py (HDL-64E 64 x 512 static sweeps every 4 m along 180 m of streets,
    leaf --leaf), places every 4 m.
Reported (GPU time from CUDA-event profiling, family "dense", median / min / max over --reps rounds after a warm-up):
  * database build against candidates (100, 1000, 10000) and rays (64 x 360, 64 x 720), max_range 100 m, ray index
    already built;
  * query against candidates (1000, 10000, 100000) with the recommended params (20 x 60);
  * wall time of dense_relocalize_global at the recommended parameters beside dense_relocalize at its recommended
    grid (14661 poses) around the truth, both for one held-out HDL-64E sweep on the route map;
  * with --ptxas, registers and spills of every place kernel from nvcc -Xptxas -v.

    python tools/dense_place_cost.py [--sweeps 55 --leaf 0.1 --reps 7 --ptxas]
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

sys.dont_write_bytecode = True
from dense_cost import ROOT, dense_ctx, gpu_info, profiled, replay_run, require_cuda, stats  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))


def ptxas():
    csrc = os.path.join(ROOT, "loam_velodyne_b200", "csrc")
    r = subprocess.run(["make", "-s", "-C", csrc, "ptxas"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    out, cur = {}, None
    for line in r.stdout.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1) if ("dense_place" in m.group(1) or "dense_raycast" in m.group(1)) else None
        elif cur and "spill" in line:
            out.setdefault(cur, {})["spills"] = line.strip()
        elif cur and "Used" in line:
            out.setdefault(cur, {})["used"] = line.split("info    :")[-1].strip()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sweeps", type=int, default=55)
    ap.add_argument("--leaf", type=float, default=0.1)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--ptxas", action="store_true")
    args = ap.parse_args()

    require_cuda("dense_place_cost")
    from loam_velodyne_b200 import api, synth
    import align_reference as ar
    from test_dense_place import route
    scene, lidar, sweeps, fulls, twists = replay_run(args.sweeps)
    c, _ = dense_ctx(fulls, args.leaf)
    n_target = c.dense_target_build(None, 2, (0.0, 0.0, 0.0))
    prm = api.PlaceParams.default()
    elev = np.linspace(lidar.lower_deg, lidar.upper_deg, lidar.n_rings)
    rng = np.random.RandomState(1)
    centre = np.asarray(twists[args.sweeps // 2][3:], np.float64)

    def positions(k):
        return np.stack([centre[0] + rng.uniform(-20, 20, k), np.full(k, centre[1]),
                         centre[2] + rng.uniform(-20, 20, k)], 1).astype(np.float32)

    def timed(ctx, fn):
        return stats(profiled(ctx, {"call": fn}, args.reps)["call"].gpu_ms)

    c.dense_raycast(api.lidar_rays(elev, 8), twists[0])  # the ray index, outside the timed builds
    build = {}
    for n_az in (360, 720):
        rays = api.lidar_rays(elev, n_az)
        for k in (100, 1000, 10000):
            p = positions(k)
            build[f"{k}_candidates_{rays.shape[0]}_rays"] = timed(c, lambda: c.dense_place_build(p, rays, prm))
    query = {}
    q = sweeps[args.sweeps // 2][0]
    for k in (1000, 10000, 100000):
        c.dense_place_build(positions(k), api.lidar_rays(elev, 360), prm)
        query[f"{k}_candidates"] = timed(c, lambda: c.dense_place_query(q, top_m=api.PLACE_TOP_M))
    c.close()

    # the route map
    small = synth.Lidar.hdl64(512)
    pos, yaw = route(4.0)
    r, _ = dense_ctx((ar.static_sweep(scene, small, np.array([0.0, yaw[k], 0.0, *pos[k]]), seed=k)[1]
                      for k in range(pos.shape[0])), args.leaf)
    n_route = r.dense_target_build(None, 2, (0.0, 0.0, 0.0))
    traj, _ = route(1.0)
    places = api.thin_trajectory(traj, api.PLACE_SPACING)
    rays = api.lidar_rays(np.linspace(small.lower_deg, small.upper_deg, small.n_rings), 360)
    r.dense_raycast(rays[:8], np.zeros(6))
    route_build = timed(r, lambda: r.dense_place_build(places, rays, prm))
    truth = np.array([0.0, 2.0, 0.0, 31.0, 0.0, 0.8], np.float32)
    qs = ar.static_sweep(scene, small, truth.astype(np.float64), seed=77)[0]
    grid = api.reloc_grid(truth)
    wall = {"global": [], "dense_relocalize_default_grid": []}
    ok = {}
    for rep in range(args.reps + 1):
        t0 = time.perf_counter()
        g = r.dense_relocalize_global(qs)
        t1 = time.perf_counter()
        d = r.dense_relocalize(qs, grid)
        t2 = time.perf_counter()
        if rep:
            wall["global"].append((t1 - t0) * 1e3)
            wall["dense_relocalize_default_grid"].append((t2 - t1) * 1e3)
        ok = {"global": ar.twist_error(g[0]["fine"][0], truth) if g else None,
              "dense_relocalize": ar.twist_error(d[0]["fine"][0], truth) if d else None}
    r.close()

    print(json.dumps({
        "workload": f"config-3 map ({args.sweeps} sweeps at leaf {args.leaf} m, {n_target} target voxels); route map "
                    f"({pos.shape[0]} HDL-64E 64 x 512 static sweeps, {n_route} target voxels, {places.shape[0]} places)",
        "params": [prm.rings, prm.sectors, prm.max_radius, prm.height_offset, prm.min_range, prm.max_range],
        "reps": args.reps, "build_gpu_ms": build, "query_gpu_ms": query, "route_build_gpu_ms": route_build,
        "relocalize_wall_ms": {k: stats(v) for k, v in wall.items()},
        "global_hypotheses": api.PLACE_TOP_M * (2 * api.PLACE_YAW_STEPS + 1) * (2 * api.PLACE_XZ_STEPS + 1) ** 2,
        "default_grid_hypotheses": int(grid.shape[0]), "error_m_deg": ok,
        "ptxas": ptxas() if args.ptxas else "not run",
        "gpu": gpu_info(),
    }))


if __name__ == "__main__":
    main()
