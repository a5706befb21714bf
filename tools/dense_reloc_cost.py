#!/usr/bin/env python
"""What relocalising a sweep in the whole-run voxel map costs.

Workload: the replayed hdl64_1m map (tools/dense_cost.py), --sweeps sweeps at --leaf, target built at normals radius
2.  Reported, with the card's name and power limit read in the same run:
  * the score pass (dense_score at radius 3): GPU time of its launches (CUDA-event profiling, family "dense") against
    k (1 k, 10 k, 100 k poses near the mapped pose) at n = 32 k points, and against n (the 131 k-point sweep strided to
    8 k, 32 k and 131 k points) at k = 10 k; median, min and max over --reps after one warm-up;
  * one batched alignment iteration (dense_align_batch, max_iterations 1, radius 3) of the 131 k-point sweep against k
    (1, 16, 256, 1024): GPU time;
  * a full relocalisation at the recommended parameters (full-circle 2 deg yaw grid, 0.4 m x-z steps four to each side
    of a prior 1.5 m off; 14661 hypotheses): host wall time and the error of candidate 0;
  * dense_align coarse to fine (radius 3, then 1, 10 iterations each) from 0.3 m / 2 deg off: host wall time of this
    library against --baseline-lib (the same entry point built from an earlier revision, target loaded from this
    library's export), the two arms alternating round by round.

    python tools/dense_reloc_cost.py [--sweeps 55 --leaf 0.1 --reps 10 --baseline-lib path/libloam_b200.so]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import sys
import time

import numpy as np

sys.dont_write_bytecode = True
from dense_cost import ROOT, dense_ctx, gpu_info, profiled, replay_run, require_cuda, stats  # noqa: E402


class BaselineAlign:
    """loam_b200_dense_align of another build of the library, on a context of its own holding a loaded target."""

    def __init__(self, path, leaf, cent, nrm):
        from loam_velodyne_b200 import api
        self.api = api
        L = self.L = C.CDLL(path)
        vp = C.c_void_p
        L.loam_b200_create.argtypes = [C.POINTER(vp), C.c_int]
        L.loam_b200_destroy.argtypes = [vp]
        L.loam_b200_dense_target_load.argtypes = [vp, C.c_float, api._F, api._F, C.c_int]
        L.loam_b200_dense_align.argtypes = [vp, api._F, C.c_int, C.c_int, C.POINTER(api.Pose), C.c_int, C.c_int,
                                            C.POINTER(api.AlignResult)]
        self.h = vp()
        assert L.loam_b200_create(C.byref(self.h), 0) == 0
        self.cent, self.nrm = np.ascontiguousarray(cent, np.float32), np.ascontiguousarray(nrm, np.float32)
        assert L.loam_b200_dense_target_load(self.h, np.float32(leaf), api._fp(self.cent), api._fp(self.nrm),
                                             self.cent.shape[0]) == 0

    def align(self, pts, twist6, radius, iters):
        a = np.ascontiguousarray(pts, np.float32)
        p = self.api.make_pose(twist6)
        r = self.api.AlignResult()
        assert self.L.loam_b200_dense_align(self.h, self.api._fp(a), a.shape[0], 0, C.byref(p), radius, iters,
                                            C.byref(r)) == 0
        return np.array(list(r.rot) + list(r.pos), np.float32), r.iterations

    def close(self):
        self.L.loam_b200_destroy(self.h)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sweeps", type=int, default=55)
    ap.add_argument("--leaf", type=float, default=0.1)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--baseline-lib", default=None)
    args = ap.parse_args()

    require_cuda("dense_reloc_cost")
    from loam_velodyne_b200 import api
    _, _, sweeps, fulls, twists = replay_run(args.sweeps)
    c, _ = dense_ctx(fulls, args.leaf)
    n_target = c.dense_target_build(None, 2, (0.0, 0.0, 0.0))

    k = args.sweeps // 2
    pts = sweeps[k][0]
    mapped = twists[k]
    rng = np.random.RandomState(5)

    def near(n):
        d = np.zeros((n, 6), np.float32)
        d[:, 1] = rng.uniform(-0.2, 0.2, n)
        d[:, 3] = rng.uniform(-1.0, 1.0, n)
        d[:, 5] = rng.uniform(-1.0, 1.0, n)
        return (mapped + d).astype(np.float32)

    def gpu_ms(fn):
        return stats(profiled(c, {"call": fn}, args.reps)["call"].gpu_ms)

    strided = {n: pts[::max(1, pts.shape[0] // n)][:n] for n in (8192, 32768, pts.shape[0])}
    poses = {kk: near(kk) for kk in (1000, 10000, 100000)}
    score_k = {f"k{kk}": gpu_ms(lambda: c.dense_score(strided[32768], poses[kk], 3)) for kk in poses}
    score_n = {f"n{n}": gpu_ms(lambda: c.dense_score(strided[n], poses[10000], 3)) for n in strided}
    batch_it = {f"k{kk}": gpu_ms(lambda: c.dense_align_batch(pts, poses[1000][:kk], 3, 1)) for kk in (1, 16, 256, 1024)}

    a = rng.uniform(0, 2 * math.pi)
    prior = (mapped + np.array([0, 1.0, 0, 1.5 * math.cos(a), 0, 1.5 * math.sin(a)], np.float32)).astype(np.float32)
    hyps = api.reloc_grid(prior, api.RELOC_YAW_STEP_DEG, None, api.RELOC_XZ_STEP, api.RELOC_XZ_STEPS)
    from align_reference import twist_error  # noqa: E402  (tests/ is on the path below)
    wall, err = [], None
    for rep in range(max(3, args.reps // 3) + 1):
        t0 = time.perf_counter()
        cands = c.dense_relocalize(pts, hyps)
        el = time.perf_counter() - t0
        if rep:
            wall.append(1e3 * el)
        err = twist_error(cands[0]["fine"][0], mapped) if cands else None

    w, u = rng.normal(size=3), rng.normal(size=3)
    init = (mapped + np.concatenate([w / np.linalg.norm(w) * math.radians(2.0), u / np.linalg.norm(u) * 0.3])
            ).astype(np.float32)
    base = None
    if args.baseline_lib:
        cent, _, nrm = c.dense_export_normals(None, 2, (0.0, 0.0, 0.0))
        base = BaselineAlign(args.baseline_lib, args.leaf, cent, nrm)
    arms = {"this": [], "baseline": []}
    same = True
    for rep in range(args.reps + 1):
        for arm in (("this", "baseline") if rep % 2 else ("baseline", "this")):
            if arm == "baseline" and base is None:
                continue
            t0 = time.perf_counter()
            if arm == "this":
                r1, _ = c.dense_align(pts, init, 3, 10)
                r2, _ = c.dense_align(pts, r1, 1, 10)
            else:
                r1, _ = base.align(pts, init, 3, 10)
                r2, _ = base.align(pts, r1, 1, 10)
            el = time.perf_counter() - t0
            if rep:
                arms[arm].append(1e3 * el)
            if arm == "this":
                mine = r2
            else:
                theirs = r2
        if base is not None:
            same = same and np.array_equal(mine.view(np.uint32), theirs.view(np.uint32))
    if base is not None:
        base.close()
    c.close()

    print(json.dumps({
        "workload": f"whole-run map of hdl64_1m (BASELINE config 3), {args.sweeps} sweeps replayed at leaf {args.leaf} m;"
                    f" sweep {k} ({pts.shape[0]} points)",
        "target_voxels": n_target, "reps": args.reps,
        "score_gpu_ms_vs_k_at_n32768_r3": score_k, "score_gpu_ms_vs_n_at_k10000_r3": score_n,
        "batch_iteration_gpu_ms_r3_n131k": batch_it,
        "relocalize_wall_ms": stats(wall), "relocalize_hypotheses": int(hyps.shape[0]),
        "relocalize_error_m_deg": err,
        "dense_align_coarse_to_fine_wall_ms": {k_: stats(v) for k_, v in arms.items() if v},
        "dense_align_same_bits_as_baseline": same if base is not None else None,
        "gpu": gpu_info(),
    }))


if __name__ == "__main__":
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    main()
