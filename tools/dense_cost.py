"""What the whole-run voxel map cost tools (tools/dense_*.py) share: the workload, the replayed run, the timing loops
and the card report.  A library, not a script.

The workload, "hdl64_1m", is BASELINE config 3: the synthetic city of synth.make_scene(), an HDL-64E (64 x 2048
points per sweep) moving through it at 5 deg of yaw per sweep, and a 1 M-point surrounding map seeded into the mapping
stage before the first sweep.  Sweep i is synth.make_sweep(scene, lidar, i), so every run sees the same sweeps.

The replay: the first --sweeps sweeps go through api.Pipeline one at a time, and after each the mapping stage's
registered full-resolution cloud (mapping.cloud("full")) and mapped pose (mapping.twist("aft")) are kept.  Those
clouds, inserted in order into a kernel-level context (api.Ctx) with the whole-run map at --leaf, make the map the
export, alignment, relocalisation, ray-cast, distance-field and place tools measure; at leaf 0.1 m and 55 sweeps it is
the "config-3 map" of DESIGN.md section 5.1.  The streaming tools run the same sweeps from HBM through the concurrent
pipeline instead.

Kernel times come from the library's CUDA-event profiling (family "dense" of profile_get).  Every tool prints one JSON
line whose "gpu" object names the card and its power limit, read in the same run.
"""
from __future__ import annotations

import math
import os
import subprocess
import sys
import time
from typing import Any, NamedTuple

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    """{"name", "power_limit_w"} of device 0: from NVML, else from nvidia-smi's read-only query, else the name alone
    from torch with power_limit_w None."""
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(0)
        name = pynvml.nvmlDeviceGetName(h)
        return {"name": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": round(pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0, 1)}
    except Exception:
        pass
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, check=True).stdout
        name, limit = out.splitlines()[0].rsplit(",", 1)
        return {"name": name.strip(), "power_limit_w": round(float(limit), 1)}
    except Exception:
        pass
    import torch
    return {"name": torch.cuda.get_device_name(0), "power_limit_w": None}


def stats(values):
    """Median, min and max, rounded to 4 decimals."""
    return {"median": round(float(np.median(values)), 4), "min": round(float(np.min(values)), 4),
            "max": round(float(np.max(values)), 4)}


def require_cuda(tool_name):
    """Exit with a message when there is no CUDA device: every number these tools report is a GPU measurement."""
    import torch
    if not torch.cuda.is_available():
        raise SystemExit(f"{tool_name}: no CUDA device (nothing here runs on the CPU)")


def hdl64_1m(n):
    """The scene, the HDL-64E, the 1 M-point seed map (corner, surf) and the first n sweeps (points, ring sizes)."""
    from loam_velodyne_b200 import synth
    scene = synth.make_scene()
    lidar = synth.Lidar.hdl64()
    seed = synth.make_map(scene, 1_000_000)
    sweeps = [synth.make_sweep(scene, lidar, i, yaw_rate=math.radians(5.0)) for i in range(n)]
    return scene, lidar, seed, sweeps


def replay_run(n):
    """The first n sweeps of hdl64_1m through api.Pipeline one at a time: (scene, lidar, sweeps, the registered
    full-resolution clouds, the mapped poses)."""
    from loam_velodyne_b200 import api
    scene, lidar, seed, sweeps = hdl64_1m(n)
    seq = api.Pipeline()
    seq.seed_map(*seed)
    fulls, twists = [], []
    for pts, rs in sweeps:
        seq.sweep(pts, rs)
        fulls.append(seq.mapping.cloud("full"))
        twists.append(seq.mapping.twist("aft"))
    seq.sync()
    del seq
    return scene, lidar, sweeps, fulls, twists


def dense_ctx(fulls, leaf):
    """A kernel-level context with the whole-run map at leaf filled from fulls in order, and its voxel count."""
    from loam_velodyne_b200 import api
    c = api.Ctx(0)
    c.dense_enable(leaf)
    for f in fulls:
        c.cloud_upload(api.C_MAP_FULL, f)
        c.dense_insert(api.C_MAP_FULL)
    return c, c.dense_stats()["voxels"]


class Profile(NamedTuple):
    gpu_ms: list        # "dense" kernel time of each timed call
    launches: int       # "dense" launches of the last call
    host_ms: list       # perf_counter around each timed call
    out: Any            # what the last call returned


def profiled(c, calls, reps):
    """Each of calls ({name: fn}) in turn, one warm-up round and then reps timed rounds, with c's profiling reset
    before every call.  Returns {name: Profile}."""
    gpu = {k: [] for k in calls}
    host = {k: [] for k in calls}
    launches, outs = {}, {}
    for rep in range(reps + 1):
        for name, fn in calls.items():
            c.profile(True)
            t0 = time.perf_counter()
            outs[name] = fn()
            el = time.perf_counter() - t0
            ms, launches[name] = c.profile_get()["dense"]
            if rep:
                gpu[name].append(ms)
                host[name].append(1e3 * el)
    return {k: Profile(gpu[k], launches[k], host[k], outs[k]) for k in calls}


def stream_windows(args, sweeps, pipeline, arms, probe=None):
    """Streaming throughput of each arm: windows of args.steps sweeps submitted from HBM, each on a fresh
    pipeline(arm) (a seeded api.Pipeline with the arm under test enabled) after args.warmup sweeps, the arms
    alternating, until every arm has args.min_seconds of timed windows and at least three, or args.max_windows
    windows.  Returns ({arm: sweeps/s median, min and max, window count, window ms min/median/max},
    {arm: [probe(p, arm) after each window]})."""
    import torch
    d_sweeps = [torch.from_numpy(pts).to("cuda:0") for pts, _ in sweeps]
    torch.cuda.synchronize()
    n = args.warmup + args.steps

    def window(arm):
        p = pipeline(arm)

        def run(lo, hi):
            got = 0
            for i in range(lo, hi):
                p.submit(ring_sizes=sweeps[i][1], device_ptr=d_sweeps[i].data_ptr())
                if p.collect(wait=False) is not None:
                    got += 1
            while got < hi - lo:
                p.collect(wait=True)
                got += 1
            p.sync()

        run(0, args.warmup)
        p.stage_seconds(reset=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run(args.warmup, n)  # ends with every stage, the map's work included, finished on the GPU
        torch.cuda.synchronize()
        el = time.perf_counter() - t0
        seen = probe(p, arm) if probe else None
        del p
        return el, seen

    windows = {a: [] for a in arms}
    probes = {a: [] for a in arms}
    while True:
        for a in arms:
            el, seen = window(a)
            windows[a].append(el)
            probes[a].append(seen)
        if all(sum(windows[a]) >= args.min_seconds and len(windows[a]) >= 3 for a in arms) or \
                len(windows[arms[-1]]) >= args.max_windows:
            break

    def rate(els):
        s = sorted(els)
        sps = [args.steps / e for e in s]
        return {"sweeps_per_s_median": round(args.steps / s[len(s) // 2], 1), "sweeps_per_s_min": round(min(sps), 1),
                "sweeps_per_s_max": round(max(sps), 1), "windows": len(s),
                "window_ms_min_median_max": [round(1e3 * s[0], 2), round(1e3 * s[len(s) // 2], 2), round(1e3 * s[-1], 2)]}

    return {a: rate(windows[a]) for a in arms}, probes
