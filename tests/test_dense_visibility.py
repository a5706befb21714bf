"""The visibility pass of the whole-run voxel map on the GPU (csrc/densemap.cuh) against its numpy restatement
(tests/visibility_reference.py): centroids, counts and hits bit for bit, misses equal except where the restatement
flags a voxel within 1e-9 of a pixel edge or of the miss threshold (CUDA's atan2 may differ from libm's in the last
ulp).  Then the mapping stage and the streaming pipeline with the pass on, and the trail of a moving box end to end."""
import dataclasses
import math

import numpy as np
import pytest

import visibility_reference as vr
from test_visibility_reference import EXPECTED, H_RES, MARGIN, RATIO, V_RES

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def assert_matches(got, ref, what, max_uncertain=None):
    """got = Ctx.dense_export(max_miss_ratio=inf, evidence=True) -> returns the number of voxels whose misses differ
    (all of them flagged by the restatement)."""
    gc, gn, gh, gm = got
    rc, rn, rh, rm = ref.export_filtered()
    assert gc.shape == rc.shape, f"{what}: {gc.shape} vs {rc.shape}"
    assert np.array_equal(gn, rn), f"{what}: counts differ"
    assert np.array_equal(bits(gc), bits(rc)), f"{what}: centroids differ"
    assert np.array_equal(gh, rh), f"{what}: hits differ"
    diff = gm != rm
    unc = np.isin(ref.keys, np.array(sorted(ref.uncertain), np.uint64))
    assert not np.any(diff & ~unc), f"{what}: {int((diff & ~unc).sum())} unflagged voxels differ in misses"
    if max_uncertain is not None:
        assert unc.sum() <= max_uncertain, f"{what}: {int(unc.sum())} voxels near an edge"
    print(f"{what}: {gc.shape[0]} voxels, {int(gm.astype(bool).sum())} with misses, {int(unc.sum())} flagged, "
          f"{int(diff.sum())} differ")
    return int(diff.sum())


@pytest.fixture(scope="module")
def runs(scene):
    from loam_velodyne_b200 import synth
    return {"vlp16": vr.moving_box_run(scene, synth.Lidar.vlp16(), 16),
            "hdl64": vr.moving_box_run(scene, synth.Lidar.hdl64(), 10)}


def tilted(twist, k):
    """The sweep's pose with some roll and pitch as well, so that all three rotations of the pass are exercised."""
    t = np.array(twist, np.float32)
    t[0] += np.float32(0.01 * (k % 3))
    t[2] -= np.float32(0.015 * (k % 4))
    return t


@pytest.mark.parametrize("lidar", ["vlp16", "hdl64"])
def test_observe_insert_sequences(build_libs, runs, lidar):
    """dense_observe + dense_insert at known poses, checked after every sweep; the table grows on the way."""
    from loam_velodyne_b200 import api
    leaf = 0.1
    ref = vr.VisibilityMapRef(leaf, h_res=0.5, v_res=1.0, margin=0.3)
    c = api.Ctx(0)
    try:
        c.dense_enable(leaf)
        c.dense_visibility(0.5, 1.0, 0.3)
        for k, (pts, twist, _) in enumerate(runs[lidar]):
            pose = tilted(twist, k)
            c.cloud_upload(api.C_MAP_FULL, pts)
            c.dense_observe(api.C_MAP_FULL, pose)
            c.dense_insert(api.C_MAP_FULL)
            ref.observe(pts, pose)
            ref.insert(pts)
            assert_matches(c.dense_export(math.inf, evidence=True), ref, f"{lidar} sweep {k}",
                           max_uncertain=ref.keys.size // 1000 + 5)
        assert int(ref.misses.astype(bool).sum()) > 100
        # the unfiltered export is the same with the evidence on; the filter is the restatement's
        plain = c.dense_export()
        full = c.dense_export(math.inf)
        assert np.array_equal(bits(plain[0]), bits(full[0])) and np.array_equal(plain[1], full[1])
        if not ref.uncertain:
            for ratio in (0.0, 0.5, 1.0):
                g = c.dense_export(ratio, evidence=True)
                r = ref.export_filtered(ratio)
                assert np.array_equal(bits(g[0]), bits(r[0])) and all(np.array_equal(a, b) for a, b in zip(g[1:], r[1:]))
    finally:
        c.close()


def test_threshold_and_wrap_edges(build_libs):
    """The strict threshold (image == r + margin: no miss; one double more: a miss), the azimuth wrap at +-180 deg and
    the row clamp at +90 deg, as in test_visibility_reference."""
    from loam_velodyne_b200 import api
    c = api.Ctx(0)
    try:
        c.dense_enable(0.1)

        def case(stored, seen, h, v, margin):
            c.dense_clear()
            c.dense_visibility(h, v, margin)
            c.cloud_upload(api.C_MAP_FULL, np.array(stored, np.float32))
            c.dense_insert(api.C_MAP_FULL)
            c.cloud_upload(api.C_MAP_FULL, np.array(seen, np.float32))
            c.dense_observe(api.C_MAP_FULL, (0, 0, 0, 0, 0, 0))
            return c.dense_export(evidence=True)[3].tolist()

        below = float(np.nextafter(5.5, 0.0)) - 5.0
        assert case([[0, 0, 5, 1]], [[0, 0, 5.5, 1]], 0.5, 0.5, 0.5) == [0]
        assert case([[0, 0, 5, 1]], [[0, 0, 5.5, 1]], 0.5, 0.5, below) == [1]
        a = math.radians(-179.9)
        assert case([[0, 0, -5, 1]], [[20 * math.sin(a), 0, 20 * math.cos(a), 1]], 1.0, 1.0, 0.2) == [1]
        e = math.radians(89.5)
        assert case([[0, 10, 0, 1]], [[0, 30 * math.sin(e), 30 * math.cos(e), 1]], 1.0, 1.0, 0.2) == [1]
    finally:
        c.close()


def test_edge_cases(build_libs, runs):
    from loam_velodyne_b200 import api
    pts = [r[0] for r in runs["vlp16"][:3]]
    tw = [r[1] for r in runs["vlp16"][:3]]
    c = api.Ctx(0)
    try:
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_visibility(1.0, 1.0, 0.5)  # no dense map
        c.dense_enable(0.2, 5000)  # a cap below one sweep's voxels: the rest is dropped, never observed
        for bad in ((float("nan"), 1, 1), (1, float("inf"), 1), (-1, 1, 1), (361, 1, 1), (1, 0, 1), (1, 181, 1),
                    (1, 1, -0.1), (0.05, 0.05, 1), (360.0 / 4097, 180.0 / 4097, 0.5)):
            with pytest.raises(api.LoamB200Error, match="invalid argument"):
                c.dense_visibility(*bad)
        c.dense_visibility(360.0 / 4096, 180.0 / 4096, 0.5)  # exactly 2^24 pixels
        c.dense_visibility(0, 0, 0)
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_observe(api.C_MAP_FULL, tw[0])  # off: observe refused
        ref = vr.VisibilityMapRef(0.2, 5000, 1.0, 2.0, 0.5)
        c.dense_visibility(1.0, 2.0, 0.5)
        empty = np.zeros((0, 4), np.float32)
        nan = np.full((1000, 4), np.nan, np.float32)
        seq = [(pts[0], tw[0]), (empty, tw[1]), (nan, tw[1]), (pts[1], tw[1])]
        for p, t in seq:
            c.cloud_upload(api.C_MAP_FULL, p)
            c.dense_observe(api.C_MAP_FULL, t)
            c.dense_insert(api.C_MAP_FULL)
            ref.sweep(p, t)
        assert ref.stats()["dropped"] > 0 and c.dense_stats() == ref.stats()
        assert_matches(c.dense_export(evidence=True), ref, "capped")
        # raise the cap: the table grows between this sweep's observe and the next, which must scan the new table
        c.dense_enable(0.2)
        ref.max_voxels = 2**31 - 1
        for p, t in [(pts[1], tw[1]), (pts[2], tw[2]), (pts[0], tw[0])]:
            c.cloud_upload(api.C_MAP_FULL, p)
            c.dense_observe(api.C_MAP_FULL, t)
            c.dense_insert(api.C_MAP_FULL)
            ref.sweep(p, t)
        assert ref.stats()["voxels"] > 2 * 5000
        assert_matches(c.dense_export(evidence=True), ref, "after growth")
        # off again: inserts still count hits, no misses
        c.dense_visibility(0.0, 0.0, 0.0)
        ref.set_visibility(0.0, 1.0, 0.0)
        c.cloud_upload(api.C_MAP_FULL, pts[2])
        c.dense_insert(api.C_MAP_FULL)
        ref.insert(pts[2])
        assert_matches(c.dense_export(evidence=True), ref, "pass off")
        with pytest.raises(api.LoamB200Error, match="invalid argument"):
            c.dense_export(float("nan"))
        c.dense_clear()
        assert c.dense_export(1.0, evidence=True)[0].shape == (0, 4)
    finally:
        c.close()
    s = api.Ctx(0)
    s.map_set_shard(0, 2)
    with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
        s.dense_visibility(1.0, 2.0, 0.5)
    s.close()


SUMS = [(0.01, 1.3, -0.02, 0.3, 0.1, 0.2), (-0.02, 2.4, 0.03, 24.9, 0.5, 24.8), (0.0, -1.1, 0.0, -74.9, 0.2, -25.1),
        (0.03, 3.0, -0.01, -380.0, 1.0, 10.0), (0.0, -2.9, 0.02, 380.0, -1.0, -30.0), (0.0, 0.4, 0.0, -5.0, 0.0, 3.0)]
SUMS += [(0.0, 0.05 * i, 0.0, 0.4 * i, 0.02 * i, 0.9 * i) for i in range(16)]


# the synthetic lidar fires on an exact 0.4 deg azimuth lattice; a pixel grid offset from it keeps returns off the pixel
# edges, so that few voxels are exempt from the exact comparison of misses
MAP_H_RES = 0.97


def mapping_run(scene, map_200k, visibility):
    """The mapping stage as test_dense_map runs it, dense map on, visibility pass on or off."""
    from loam_velodyne_b200 import api, synth
    reg = api.ScanRegistration()
    m = api.LaserMapping(0.1, 10)
    m.seed(*map_200k)
    m.enable_dense_map(0.1)
    if visibility:
        m.enable_dense_visibility(MAP_H_RES, V_RES, MARGIN)
    lidar = synth.Lidar.vlp16(n_az=900)
    outs, fulls, poses = [], [], []
    for it, sum6 in enumerate(SUMS):
        pts, rs = synth.make_sweep(scene, lidar, it, yaw_rate=math.radians(5.0))
        reg.process(pts, rs)
        m.set_inputs(reg.cloud("less_sharp"), reg.cloud("less_flat"), pts)
        m.update_odometry(np.asarray(sum6, np.float32))
        assert m.process()
        full = m.cloud("full")
        fulls.append(full)
        poses.append(m.twist("tobe"))
        outs.append((m.twist("aft"), m.twist("bef"), m.twist("tobe"), full, m.cloud("surf_stack_ds")))
    outs.append((m.cloud("corner_cubes"), m.cloud("surf_cubes")))
    return outs, fulls, poses, m


def test_mapping_stage(build_libs, scene, map_200k):
    off, _, _, m_off = mapping_run(scene, map_200k, False)
    on, fulls, poses, m = mapping_run(scene, map_200k, True)
    for i, (a, b) in enumerate(zip(off, on)):
        for x, y in zip(a, b):
            assert np.array_equal(bits(x), bits(y)), f"sweep {i}: an output changed with the visibility pass on"
    a, b = m_off.dense_map(), m.dense_map()
    assert np.array_equal(bits(a[0]), bits(b[0])) and np.array_equal(a[1], b[1])
    assert np.array_equal(m_off.dense_map(evidence=True)[3], np.zeros_like(a[1], np.uint16))
    ref = vr.VisibilityMapRef(0.1, h_res=MAP_H_RES, v_res=V_RES, margin=MARGIN)
    for pts, pose in zip(fulls, poses):
        ref.sweep(pts, pose)
    assert int(ref.misses.astype(bool).sum()) > 100
    assert_matches(m.dense_map(evidence=True), ref, "mapping stage", max_uncertain=ref.keys.size // 1000 + 5)
    kept = m.dense_map(RATIO)
    assert kept[0].shape[0] < a[0].shape[0]


def pow2_slots(voxels):
    """Table slots the host sizes for an upper bound of `voxels` (load factor <= 0.5, at least 1024)."""
    s = 1024
    while s < 2 * voxels:
        s *= 2
    return s


def test_streaming_pipeline(build_libs, scene, map_200k):
    """The streaming pipeline gives the sequential chain's evidence, and with the pass on the table is sized from the
    voxels stored, as with it off (the pass must not hide the insertion's completion from the table sizing)."""
    from loam_velodyne_b200 import api, synth
    lidar = synth.Lidar.vlp16()
    sweeps = [synth.make_sweep(scene, lidar, i, yaw_rate=math.radians(5.0)) for i in range(12)]
    got, slots = {}, {}
    for vis, stream in ((False, True), (True, False), (True, True)):
        p = api.Pipeline()
        p.seed_map(*map_200k)
        p.mapping.enable_dense_map(0.1)
        if vis:
            p.mapping.enable_dense_visibility(H_RES, V_RES, MARGIN)
        if stream:
            p.run_stream(sweeps)
        else:
            for pts, rs in sweeps:
                p.sweep(pts, rs)
        got[vis, stream] = p.mapping.dense_map(evidence=True)
        slots[vis, stream] = p.mapping.dense_table_slots()
    a, b = got[True, False], got[True, True]
    assert a[0].shape[0] > 10000 and int(a[3].astype(bool).sum()) > 0
    assert np.array_equal(bits(a[0]), bits(b[0]))
    for x, y in zip(a[1:], b[1:]):
        assert np.array_equal(x, y)
    off = got[False, True]
    assert np.array_equal(bits(off[0]), bits(a[0])) and np.array_equal(off[1], a[1]) and np.array_equal(off[2], a[2])
    # at most the running bound of one sweep in flight above the stored voxels
    most = pow2_slots(a[0].shape[0] + 2 * max(p.shape[0] for p, _ in sweeps))
    print(f"table slots: off {slots[False, True]}, on {slots[True, False]} / {slots[True, True]}, bound {most}")
    for k, v in slots.items():
        assert 0 < v <= most, f"{k}: {v} table slots for {a[0].shape[0]} voxels"


def test_pipeline_removes_moving_box_trail(build_libs, scene, map_200k):
    """The whole pipeline (estimated poses) over the street with the box driving across: the trail goes, the static map
    stays, at the rates the ground-truth restatement pins.  Voxels are classified by where their centroid lies."""
    from loam_velodyne_b200 import api, synth
    lidar = synth.Lidar.vlp16()
    n = 24
    boxes = [vr.box_at(k) for k in range(n)]
    p = api.Pipeline()
    p.seed_map(*map_200k)
    p.mapping.enable_dense_map(0.2)
    p.mapping.enable_dense_visibility(H_RES, V_RES, MARGIN)
    for k in range(n):
        sc = dataclasses.replace(scene, boxes=np.vstack([scene.boxes, boxes[k][None, :]]))
        p.sweep(*synth.make_sweep(sc, lidar, k, yaw_rate=math.radians(5.0)))
    c, _, hits, misses = p.mapping.dense_map(evidence=True)

    def inside(ks, e):
        m = np.zeros(c.shape[0], bool)
        for b in (boxes[k] for k in ks):
            m |= ((c[:, 0] > b[0] - e) & (c[:, 0] < b[1] + e) & (c[:, 1] > b[2] - e) & (c[:, 1] < b[3] + e) &
                  (c[:, 2] > b[4] - e) & (c[:, 2] < b[5] + e))
        return m

    trail = inside(range(n - 6), 0.1) & ~inside(range(n - 6, n), 0.6) & (c[:, 1] > -1.5)
    static = ~inside(range(n), 0.6)
    keep = misses.astype(np.float64) <= RATIO * hits.astype(np.float64)
    assert p.mapping.dense_map(RATIO)[0].shape[0] == int(keep.sum())
    removed, kept = 1.0 - keep[trail].mean(), keep[static].mean()
    print(f"pipeline: {int(trail.sum())} trail voxels, removed {removed:.4f}; {int(static.sum())} static, kept {kept:.4f}")
    assert trail.sum() > 300
    assert removed >= EXPECTED["vlp16"][0] and kept >= EXPECTED["vlp16"][1]
