#!/usr/bin/env python
"""What the ground of the whole-run voxel map costs.

Workload: the replayed hdl64_1m map (tools/dense_cost.py), --sweeps sweeps at --leaf, and the target built from it
(radius 2).  Reported, with the card's name and power limit read in the same run:
  * the ground patches (loam_b200_dense_ground, default parameters, labels downloaded), with the ground's voxels;
  * the segmentation above the ground (loam_b200_dense_segment_above_ground) at tol = 0.15, 0.2 and 0.4 m, with the
    largest above-ground segment (the plain dense_segment's largest, the ground and what touches it, for comparison);
  * the ground points of the run's first HDL-64E sweep at its mapped pose (loam_b200_dense_ground_cloud), the sweep
    and the non-ground output in device memory;
each called in turn, one warm-up round and then --reps timed rounds: GPU time (CUDA-event profiling, family "dense"),
median, min and max; host wall time of the synchronous call; launches.

    python tools/dense_ground_cost.py [--sweeps 55 --leaf 0.1 --reps 10]
"""
from __future__ import annotations

import argparse
import json
import sys

sys.dont_write_bytecode = True
from dense_cost import dense_ctx, gpu_info, profiled, replay_run, require_cuda, stats  # noqa: E402

TOLS = (0.15, 0.2, 0.4)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sweeps", type=int, default=55)
    ap.add_argument("--leaf", type=float, default=0.1)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()

    require_cuda("dense_ground_cost")
    import numpy as np
    import torch
    _, _, sweeps, fulls, poses = replay_run(args.sweeps)
    c, voxels = dense_ctx(fulls, args.leaf)
    n_target = c.dense_target_build(None, 2, (0.0, 0.0, 0.0))
    plain = {t: int(c.dense_segment(t)[1]["size"][:1].sum()) for t in TOLS}
    lab, patches = c.dense_ground()
    ground_voxels = int((lab >= 0).sum())
    pts = sweeps[0][0]
    dev = torch.from_numpy(pts).cuda()
    out = torch.empty_like(dev)
    torch.cuda.synchronize()
    pose = np.asarray(poses[0], np.float32)

    calls = {"ground": lambda: c.dense_ground()}
    calls.update({f"above_tol_{t}": (lambda t=t: c.dense_segment_above_ground(t)) for t in TOLS})
    calls["ground_cloud"] = lambda: c.dense_ground_cloud(dev.data_ptr(), pose, on_device=True, n=pts.shape[0],
                                                         out=out.data_ptr())
    prof = profiled(c, calls, args.reps)
    cases = {k: {"gpu_ms": stats(p.gpu_ms), "host_ms": stats(p.host_ms), "launches": p.launches}
             for k, p in prof.items()}
    cases["ground"]["patches"] = int(prof["ground"].out[1]["size"].size)
    for t in TOLS:
        seg = prof[f"above_tol_{t}"].out[1]
        cases[f"above_tol_{t}"].update({"segments": int(seg["size"].size), "largest": int(seg["size"][:1].sum()),
                                        "largest_without_ground_removal": plain[t]})
    cl = prof["ground_cloud"].out[0]
    cases["ground_cloud"].update({"ground_points": int((cl == 1).sum()), "other_points": int((cl == 0).sum())})
    c.close()

    print(json.dumps({
        "workload": f"whole-run map of hdl64_1m (BASELINE config 3), {args.sweeps} sweeps replayed at leaf {args.leaf} m;"
                    f" cloud: its first HDL-64E sweep in device memory at its mapped pose",
        "voxels": voxels, "target_voxels": n_target, "ground_voxels": ground_voxels, "cloud_points": int(pts.shape[0]),
        "reps": args.reps, "cases": cases, "gpu": gpu_info(),
    }))


if __name__ == "__main__":
    main()
