#!/usr/bin/env python
"""What the normals of the whole-run voxel map cost at export.

Workload: the replayed hdl64_1m map (tools/dense_cost.py), --sweeps sweeps at --leaf.  Then, alternating and repeated
--reps times after one warm-up round, the filtered export (dense_export at ratio +inf) and the export with normals at
radius 1, 2 and 3: the host time of each synchronous call (perf_counter around it) and the GPU time of its kernels
(CUDA-event profiling, family "dense", reset before each call).  Prints one JSON line with medians, min and max, the
voxel count, and the card's name and power limit read in the same run.

    python tools/dense_normals_cost.py [--sweeps 55 --leaf 0.1 --reps 15]
"""
from __future__ import annotations

import argparse
import json
import math
import sys

import numpy as np

sys.dont_write_bytecode = True
from dense_cost import dense_ctx, gpu_info, profiled, replay_run, require_cuda, stats  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sweeps", type=int, default=55)
    ap.add_argument("--leaf", type=float, default=0.1)
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()

    require_cuda("dense_normals_cost")
    _, _, _, fulls, _ = replay_run(args.sweeps)
    c, voxels = dense_ctx(fulls, args.leaf)

    arms = {"filtered": lambda: c.dense_export(math.inf)}
    for r in (1, 2, 3):
        arms[f"normals_r{r}"] = (lambda r=r: c.dense_export_normals(math.inf, r, (0.0, 0.0, 0.0)))
    prof = profiled(c, arms, args.reps)
    c.close()

    out = {
        "workload": f"whole-run map of hdl64_1m (BASELINE config 3), {args.sweeps} sweeps replayed at leaf {args.leaf} m",
        "voxels": voxels, "reps": args.reps,
        "host_ms_per_call": {k: stats(p.host_ms) for k, p in prof.items()},
        "gpu_ms_per_call": {k: stats(p.gpu_ms) for k, p in prof.items()},
        "normals_gpu_ms_over_filtered_median": {
            k: round(float(np.median(prof[k].gpu_ms) - np.median(prof["filtered"].gpu_ms)), 4)
            for k in arms if k != "filtered"},
        "launches_per_call": {k: p.launches for k, p in prof.items()},
        "undefined_normals": {k: int(np.isnan(p.out[2][:, 0]).sum()) for k, p in prof.items() if k != "filtered"},
        "gpu": gpu_info(),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
