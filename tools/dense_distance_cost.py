#!/usr/bin/env python
"""What the distance field of the whole-run voxel map costs.

Workload: the replayed hdl64_1m map (tools/dense_cost.py), --sweeps sweeps at --leaf, and the target built from it
(radius 2).  Reported, with the card's name and power limit read in the same run:
  * field builds (kept on the device, no download) of a 40 x 40 x 8 m and a 100 x 100 x 12 m box centred on the last
    mapped pose at max_distance 2 m and 5 m, alternating round by round, --reps rounds after one warm-up: GPU time
    (CUDA-event profiling, family "dense"), median, min and max; cells/s of the box; the algorithmic bytes (the
    grids' reads and writes of the three passes, Meijster's stacks excluded) and their rate against 3.35 TB/s.  A box
    whose padded grid exceeds the limits is reported as refused;
  * queries with the gradient at 10^6 and 1.6 * 10^7 device-resident points spread over the first box: kernel time
    and points/s;
  * the field's device bytes.

    python tools/dense_distance_cost.py [--sweeps 55 --leaf 0.1 --reps 10]
"""
from __future__ import annotations

import argparse
import json
import math
import sys

import numpy as np

sys.dont_write_bytecode = True
from dense_cost import dense_ctx, gpu_info, profiled, replay_run, require_cuda, stats  # noqa: E402

HBM_TBPS = 3.35  # H100 SXM HBM3 peak


def algorithmic_bytes(dims, pad):
    nx, ny, nz = (int(d) for d in dims)
    nxp, nyp, nzp = nx + 2 * pad, ny + 2 * pad, nz + 2 * pad
    x_pass = 12 * nxp * nyp * nzp                     # write the left sites, read them back, write g
    y_pass = 4 * nx * nyp * nzp + 4 * nx * ny * nzp   # read g on the box's x lines, write the box's y rows
    z_pass = 4 * nx * ny * nzp + 4 * nx * ny * nz     # read them, write sq
    return x_pass + y_pass + z_pass


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sweeps", type=int, default=55)
    ap.add_argument("--leaf", type=float, default=0.1)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()

    require_cuda("dense_distance_cost")
    import torch
    from loam_velodyne_b200 import api
    _, _, _, fulls, twists = replay_run(args.sweeps)
    c, voxels = dense_ctx(fulls, args.leaf)
    n_target = c.dense_target_build(None, 2, (0.0, 0.0, 0.0))
    centre = np.asarray(twists[-1][3:], np.float64)

    boxes = {"40x40x8m": (20.0, 4.0, 20.0), "100x100x12m": (50.0, 6.0, 50.0)}
    cases, refused = {}, {}
    for bname, half in boxes.items():
        lo, dims = api.voxel_box(centre - half, centre + half, args.leaf)
        for md in (2.0, 5.0):
            name = f"{bname}_{md:g}m"
            pad = int(math.floor(float(np.float32(md)) / float(np.float32(args.leaf)))) + 1
            padded = [int(d) + 2 * pad for d in dims]
            try:
                c.dense_distance_field(lo, dims, md, download=False)
                cases[name] = (lo, dims, md, pad)
            except api.LoamB200Error as e:
                refused[name] = {"dims": [int(d) for d in dims], "padded": padded,
                                 "padded_cells": int(np.prod(padded)), "error": str(e)}
    times = profiled(c, {name: (lambda lo=lo, dims=dims, md=md: c.dense_distance_field(lo, dims, md, download=False))
                         for name, (lo, dims, md, _) in cases.items()}, args.reps)
    builds = {}
    for name, (lo, dims, md, pad) in cases.items():
        med = float(np.median(times[name].gpu_ms))
        cells = int(np.prod(dims))
        nbytes = algorithmic_bytes(dims, pad)
        builds[name] = {"dims": [int(d) for d in dims], "pad": pad, "cells": cells, "gpu_ms": stats(times[name].gpu_ms),
                        "cells_per_s": round(cells / (med * 1e-3), 1), "algorithmic_bytes": nbytes,
                        "algorithmic_tb_per_s": round(nbytes / (med * 1e-3) / 1e12, 3),
                        "fraction_of_hbm": round(nbytes / (med * 1e-3) / 1e12 / HBM_TBPS, 3)}

    first = next(iter(cases))
    lo, dims, md, _ = cases[first]
    c.dense_distance_field(lo, dims, md, download=False)
    field_bytes = c.dense_distance_bytes()
    L = float(np.float32(args.leaf))
    lo_m = torch.tensor(np.asarray(lo, np.float64) * L, dtype=torch.float32, device="cuda")
    ext_m = torch.tensor(np.asarray(dims, np.float64) * L, dtype=torch.float32, device="cuda")
    queries = {}
    for n in (1_000_000, 16_000_000):
        g = torch.Generator(device="cuda").manual_seed(n)
        pts = torch.zeros((n, 4), dtype=torch.float32, device="cuda")
        pts[:, :3] = lo_m + torch.rand((n, 3), generator=g, device="cuda") * ext_m
        torch.cuda.synchronize()
        q = profiled(c, {"query": lambda: c.dense_distance_query(pts.data_ptr(), on_device=True, n=n, gradient=True)},
                     args.reps)["query"]
        med = float(np.median(q.gpu_ms))
        queries[str(n)] = {"gpu_ms": stats(q.gpu_ms), "points_per_s": round(n / (med * 1e-3), 1),
                           "defined_fraction": round(float(np.isfinite(q.out[0]).mean()), 4)}
        del pts, q
    c.close()

    print(json.dumps({
        "workload": f"whole-run map of hdl64_1m (BASELINE config 3), {args.sweeps} sweeps replayed at leaf {args.leaf} m,"
                    f" target radius 2; boxes centred on sweep {args.sweeps - 1}'s mapped pose",
        "voxels": voxels, "target_voxels": n_target, "reps": args.reps, "builds": builds, "refused": refused,
        "queries_with_gradient": queries, "query_box": first, "field_bytes": field_bytes, "gpu": gpu_info(),
    }))


if __name__ == "__main__":
    main()
