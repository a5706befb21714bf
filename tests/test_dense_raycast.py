"""Ray casting the whole-run voxel map on the GPU (csrc/densemap.cuh: dense_raycast_kernel; loam_b200_dense_raycast)
against the numpy restatement (tests/raycast_reference.py), range bits and indices: the hand-made cases, targets built
on the GPU at three leaves from two sensors, several poses and range pairs, lidar_rays grids and a sweep's own points;
host and device input, built and loaded targets, the lazy ray index, snapshot semantics, the error paths, the
drop-in path and the mapping stage's own map."""
import math

import numpy as np
import pytest

import align_reference as ar
import raycast_reference as rr
from test_align_reference import HELD_OUT, lidars
from test_dense_align import map_ctx

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def drv(build_libs):
    from oracle import pydriver
    return pydriver.best()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def assert_cast(cast_fn, tgt, rays, twist, mn, mx, what):
    got = cast_fn(rays, twist, mn, mx)
    want = rr.cast(tgt, rays, twist, mn, mx)
    assert np.array_equal(got[1], want[1]), f"{what}: {int((got[1] != want[1]).sum())} of {rays.shape[0]} indices differ"
    assert np.array_equal(bits(got[0]), bits(want[0])), f"{what}: {int((bits(got[0]) != bits(want[0])).sum())} ranges differ"
    return got


def grid(lidar, n_az):
    from loam_velodyne_b200 import api
    return api.lidar_rays(np.linspace(lidar.lower_deg, lidar.upper_deg, lidar.n_rings), n_az)


@pytest.mark.parametrize("name", list(rr.edge_cases()))
def test_edge_cases(build_libs, name):
    """The hand-made cases, loaded into a context without the map."""
    from loam_velodyne_b200 import api
    cent, nrm, rays, twist, mn, mx, expect, _ = rr.edge_cases()[name]
    tgt = ar.loaded_target(rr.LEAF, cent, nrm)
    c = api.Ctx(0)
    try:
        c.dense_target_load(rr.LEAF, cent, nrm)
        got = assert_cast(c.dense_raycast, tgt, rays, twist, mn, mx, name)
        assert got[1].tolist() == [rr.voxel_index(tgt, e) for e in expect]
    finally:
        c.close()


# (pose, (min_range, max_range)): zero, near the held-out sweep, rotated, at negative coordinates, at a brick corner
POSES = [(np.zeros(6, np.float32), (0.0, 100.0)),
         (HELD_OUT[1], (1.5, 25.0)),
         (np.array([0.3, -1.2, 0.2, 2.0, 0.4, 5.0], np.float32), (0.0, 100.0)),
         (np.array([-0.05, 2.5, 0.1, -3.3, 0.5, -7.9], np.float32), (0.7, 60.0)),
         (np.array([0.0, 0.7, 0.0, -1.6, 0.8, 2.4], np.float32), (0.0, 400.0))]


@pytest.mark.parametrize("leaf", [0.1, 0.2, 0.4])
@pytest.mark.parametrize("sensor", ["vlp16", "hdl64"])
def test_built_targets(build_libs, scene, drv, sensor, leaf):
    """Targets built on the GPU; a lidar_rays grid from every pose and range pair, and a held-out sweep's own points."""
    lidar = lidars()[sensor]
    c, ref = map_ctx(scene, lidar, leaf)
    try:
        vp = (0.5, 1.0, -2.0)
        n = c.dense_target_build(None, 2, vp)
        tgt = ar.built_target(ref, 2, vp, drv)
        assert n == tgt.keys.size
        rays = grid(lidar, 256)
        for twist, (mn, mx) in POSES:
            r, _ = assert_cast(c.dense_raycast, tgt, rays, twist, mn, mx, f"{sensor} leaf {leaf} {twist} {mn} {mx}")
        pts = ar.static_sweep(scene, lidar, HELD_OUT[1].astype(np.float64), seed=60)[0]
        pts[::501, 1] = np.nan
        r, _ = assert_cast(c.dense_raycast, tgt, pts, HELD_OUT[1], 0.0, 100.0, f"{sensor} leaf {leaf} sweep")
        assert np.isfinite(r).mean() > 0.3  # the held-out pose sees much the map's four sweeps never saw
    finally:
        c.close()


def test_sources_targets_and_index(build_libs, scene):
    """Host and device rays give the same bits; a built target and the load of its export (into a context with the
    map off) give the same bits; the lazy index is built by the first cast and rebuilt after a load or build of a
    different map; inserts after the build change nothing; launches count under the dense family."""
    import torch
    from loam_velodyne_b200 import api, synth
    lidar = lidars()["hdl64"]
    c, _ = map_ctx(scene, lidar, 0.2)
    f = api.Ctx(0)
    try:
        vp = (0.0, 0.0, 0.0)
        c.dense_target_build(1.0, 2, vp)
        assert c.dense_ray_index_bytes() == 0
        rays = grid(lidar, 512)
        tw = HELD_OUT[2]
        c.profile(True)
        first = c.dense_raycast(rays, tw, 0.0, 80.0)
        prof = c.profile_get()
        assert prof["dense"][1] >= 4 and sum(v[1] for k, v in prof.items() if k != "dense") == 0
        assert c.dense_ray_index_bytes() > 0
        c.profile(True)
        before = c.launch_count()
        again = c.dense_raycast(rays, tw, 0.0, 80.0)
        assert c.launch_count() - before == 1 and c.profile_get()["dense"][1] == 1
        assert np.array_equal(bits(again[0]), bits(first[0])) and np.array_equal(again[1], first[1])
        dev = torch.from_numpy(rays).cuda()
        on_dev = c.dense_raycast(dev.data_ptr(), tw, 0.0, 80.0, on_device=True, n=rays.shape[0])
        torch.cuda.synchronize()
        assert np.array_equal(bits(on_dev[0]), bits(first[0])) and np.array_equal(on_dev[1], first[1])
        cent, _, nrm = c.dense_export_normals(1.0, 2, vp)
        f.dense_target_load(0.2, cent[::-1], nrm[::-1])
        loaded = f.dense_raycast(rays, tw, 0.0, 80.0)
        assert np.array_equal(bits(loaded[0]), bits(first[0])) and np.array_equal(loaded[1], first[1])
        # snapshot: an insert after the build changes nothing until the next build
        extra = ar.static_sweep(scene, synth.Lidar.hdl64(512), HELD_OUT[2].astype(np.float64) + 0.5, seed=7)[1]
        c.cloud_upload(api.C_MAP_FULL, extra)
        c.dense_insert(api.C_MAP_FULL)
        snap = c.dense_raycast(rays, tw, 0.0, 80.0)
        assert np.array_equal(bits(snap[0]), bits(first[0])) and np.array_equal(snap[1], first[1])
        # a different map replaces the index
        ecent, enrm, erays, etw, emn, emx, _, _ = rr.edge_cases()["corner"]
        c.dense_target_load(rr.LEAF, ecent, enrm)
        assert c.dense_ray_index_bytes() == 0
        e = c.dense_raycast(erays, etw, emn, emx)
        want = rr.cast(ar.loaded_target(rr.LEAF, ecent, enrm), erays, etw, emn, emx)
        assert np.array_equal(bits(e[0]), bits(want[0])) and np.array_equal(e[1], want[1])
        c.dense_target_build(1.0, 2, vp)
        rebuilt = c.dense_raycast(rays, tw, 0.0, 80.0)
        assert not np.array_equal(rebuilt[1], first[1])  # the extra sweep is in this target
        cent2, _, nrm2 = c.dense_export_normals(1.0, 2, vp)
        f.dense_target_load(0.2, cent2, nrm2)
        assert np.array_equal(bits(f.dense_raycast(rays, tw, 0.0, 80.0)[0]), bits(rebuilt[0]))
    finally:
        c.close()
        f.close()


def test_errors(build_libs, scene):
    import ctypes as C
    from loam_velodyne_b200 import api, synth
    rays = grid(lidars()["vlp16"], 64)
    c = api.Ctx(0)
    try:
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_raycast(rays, np.zeros(6))  # no target
        c.dense_target_load(0.5, np.zeros((0, 4), np.float32), np.zeros((0, 4), np.float32))
        before = c.launch_count()
        r, i = c.dense_raycast(rays, np.zeros(6))  # empty target: no hits, nothing launched
        assert np.isinf(r).all() and (i == -1).all() and c.launch_count() == before
        cent, nrm, _, _, _, _, _, _ = rr.edge_cases()["corner"]
        c.dense_target_load(rr.LEAF, cent, nrm)
        before = c.launch_count()
        r, i = c.dense_raycast(rays[:0], np.zeros(6))
        assert r.size == 0 and c.launch_count() == before
        for tw, mn, mx in ((np.zeros(6), -1.0, 10.0), (np.zeros(6), 5.0, 5.0), (np.zeros(6), 6.0, 5.0),
                           (np.zeros(6), float("nan"), 5.0), (np.zeros(6), 0.0, float("inf")),
                           (np.zeros(6), 0.0, 65536 * 0.5 * 1.001), (np.array([np.nan, 0, 0, 0, 0, 0]), 0.0, 5.0),
                           (np.array([0, 0, 0, 0, np.inf, 0]), 0.0, 5.0), (np.array([0, 0, 0, 6e5, 0, 0]), 0.0, 5.0),
                           (np.array([0, 0, 0, 0, 0, -524288.5]), 0.0, 5.0)):
            with pytest.raises(api.LoamB200Error, match="invalid argument"):
                c.dense_raycast(rays, tw, mn, mx)
        c.dense_raycast(rays, np.zeros(6), 0.0, 65536 * 0.5)  # the largest max_range at this leaf
        L = c.L
        p = api.make_pose(np.zeros(6))
        out = np.zeros(rays.shape[0], np.float32)
        assert L.loam_b200_dense_raycast(c.h, None, 10, 0, C.byref(p), 0.0, 5.0, api._fp(out), None) == -1
        assert L.loam_b200_dense_raycast(c.h, api._fp(rays), 10, 0, C.byref(p), 0.0, 5.0, None, None) == -1
        assert L.loam_b200_dense_raycast(c.h, api._fp(rays), 10, 0, None, 0.0, 5.0, api._fp(out), None) == -1
        assert L.loam_b200_dense_raycast(c.h, api._fp(rays), 10, 0, C.byref(p), 0.0, 5.0, api._fp(out), None) == 0
    finally:
        c.close()
    lidar = synth.Lidar.vlp16()
    sweeps = [synth.make_sweep(scene, lidar, i, yaw_rate=math.radians(5.0)) for i in range(3)]
    pl = api.Pipeline()
    pl.mapping.enable_dense_map(0.1)
    for q, rs in sweeps:
        pl.submit(q, rs)
    with pytest.raises(api.LoamB200Error, match="in flight"):
        pl.mapping.raycast_dense_target(rays, np.zeros(6))
    while pl.collect(wait=True) is not None:
        pass
    assert pl.mapping.build_dense_target() > 0
    r, _ = pl.mapping.raycast_dense_target(rays, np.zeros(6))
    assert np.isfinite(r).any()
    pl.sync()


SUMS = [(0.0, 0.05 * i, 0.0, 0.4 * i, 0.02 * i, 0.9 * i) for i in range(12)]
# The mapping stage's map seen from a mapped pose: the share of the sweep's rays with a hit, and |measured - cast| over
# them.  Measured with the restatement on the exported target (the GPU equals it bit for bit): sweep 3 84.2 % hit,
# median 0.021 m, 95th percentile 0.23 m; sweep 8 84.3 %, 0.042 m, 0.36 m (the sweeps are not de-skewed, and rays
# that graze the ground stop at the exit of the first ground voxel).  The bars leave about a quarter.
MAP_HIT, MAP_MEDIAN_M, MAP_P95_M = 0.8, 0.055, 0.45


def test_mapping_stage(build_libs, scene, map_200k):
    """VLP-16 through the mapping stage with the dense map on: sweep k's own points cast from transformAftMapped land
    close to their measured ranges; the drop-in path equals the Ctx path (target loaded from the export) bit for bit,
    and both equal the restatement."""
    from loam_velodyne_b200 import api, synth
    reg = api.ScanRegistration()
    m = api.LaserMapping(0.1, 10)
    m.seed(*map_200k)
    m.enable_dense_map(0.1)
    lidar = synth.Lidar.vlp16(n_az=900)
    clouds, afts = [], []
    for it, sum6 in enumerate(SUMS):
        pts, rs = synth.make_sweep(scene, lidar, it, yaw_rate=math.radians(5.0))
        reg.process(pts, rs)
        m.set_inputs(reg.cloud("less_sharp"), reg.cloud("less_flat"), pts)
        m.update_odometry(np.asarray(sum6, np.float32))
        assert m.process()
        clouds.append(pts)
        afts.append(m.twist("aft"))
    vp = (0.0, 0.0, 0.0)
    n = m.build_dense_target(None, 2, vp)
    cent, _, nrm = m.dense_map_normals(None, 2, vp)
    assert n == cent.shape[0] > 10000
    tgt = ar.loaded_target(0.1, cent, nrm)
    c = api.Ctx(0)
    try:
        c.dense_target_load(0.1, cent, nrm)
        stats = []
        for k in (3, 8):
            got = assert_cast(m.raycast_dense_target, tgt, clouds[k], afts[k], 0.0, 100.0, f"sweep {k}")
            want = c.dense_raycast(clouds[k], afts[k], 0.0, 100.0)
            assert np.array_equal(bits(got[0]), bits(want[0])) and np.array_equal(got[1], want[1])
            meas = np.linalg.norm(clouds[k][:, :3].astype(np.float64), axis=1)
            hit = np.isfinite(got[0])
            e = np.abs(got[0][hit] - meas[hit])
            stats.append((k, hit.mean(), np.median(e), np.percentile(e, 95)))
            print(f"sweep {k}: {hit.mean():.4f} hit, median {np.median(e):.4f} m, p95 {np.percentile(e, 95):.4f} m")
        for k, h, med, p95 in stats:
            assert h >= MAP_HIT and med <= MAP_MEDIAN_M and p95 <= MAP_P95_M, (k, h, med, p95)
    finally:
        c.close()
