#!/usr/bin/env python
"""What the Euclidean segmentation of the whole-run voxel map and of sweeps costs.

Workload: the replayed hdl64_1m map (tools/dense_cost.py), --sweeps sweeps at --leaf, and the target built from it
(radius 2).  Reported, with the card's name and power limit read in the same run:
  * target segmentation (loam_b200_dense_segment, labels downloaded) at tol = 0.15, 0.2 and 0.4 m;
  * cloud segmentation (loam_b200_cloud_segment) of the run's first HDL-64E sweep, device-resident, at tol = 0.3,
    0.5 and 2 m (a cloud is keyed at cell = tol, so at 2 m the voxels near the sensor hold thousands of points and the
    union pass grows with their square);
each called in turn, one warm-up round and then --reps timed rounds: GPU time (CUDA-event profiling, family "dense"),
median, min and max; host wall time of the synchronous call; launches; the number of segments.

    python tools/dense_segment_cost.py [--sweeps 55 --leaf 0.1 --reps 10]
"""
from __future__ import annotations

import argparse
import json
import sys

sys.dont_write_bytecode = True
from dense_cost import dense_ctx, gpu_info, profiled, replay_run, require_cuda, stats  # noqa: E402

TARGET_TOLS = (0.15, 0.2, 0.4)
CLOUD_TOLS = (0.3, 0.5, 2.0)  # 2 m: many points per voxel near the sensor (the quadratic case)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sweeps", type=int, default=55)
    ap.add_argument("--leaf", type=float, default=0.1)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()

    require_cuda("dense_segment_cost")
    import torch
    _, _, sweeps, fulls, _ = replay_run(args.sweeps)
    c, voxels = dense_ctx(fulls, args.leaf)
    n_target = c.dense_target_build(None, 2, (0.0, 0.0, 0.0))
    pts = sweeps[0][0]
    dev = torch.from_numpy(pts).cuda()
    torch.cuda.synchronize()

    calls = {f"target_tol_{t}": (lambda t=t: c.dense_segment(t)) for t in TARGET_TOLS}
    calls.update({f"cloud_tol_{t}": (lambda t=t: c.segment_cloud(dev.data_ptr(), t, on_device=True, n=pts.shape[0]))
                  for t in CLOUD_TOLS})
    prof = profiled(c, calls, args.reps)
    cases = {k: {"gpu_ms": stats(p.gpu_ms), "host_ms": stats(p.host_ms), "launches": p.launches,
                 "segments": int(p.out[1]["size"].size), "largest": int(p.out[1]["size"][:1].sum())}
             for k, p in prof.items()}
    c.close()

    print(json.dumps({
        "workload": f"whole-run map of hdl64_1m (BASELINE config 3), {args.sweeps} sweeps replayed at leaf {args.leaf} m;"
                    f" cloud: its first HDL-64E sweep in device memory",
        "voxels": voxels, "target_voxels": n_target, "cloud_points": int(pts.shape[0]), "reps": args.reps,
        "cases": cases, "gpu": gpu_info(),
    }))


if __name__ == "__main__":
    main()
