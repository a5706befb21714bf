"""Carve mode of the visibility pass on the GPU (csrc/densemap.cuh: dense_carve_kernel and the live occupancy index)
against its numpy restatement (tests/carve_reference.py): centroids, counts, hits and misses bit for bit -- the walk
has no transcendental function, so no voxel is exempt.  Then the index against a fresh build, the mode rules, the
errors, launch counts, the mapping stage and the drop-in path."""
import math

import numpy as np
import pytest

import carve_reference as cr
import dense_reference as dr
import visibility_reference as vr
from test_dense_visibility import SUMS, bits, tilted

pytestmark = pytest.mark.gpu


def assert_same(got, ref, what):
    """got = Ctx.dense_export(evidence=True): every field equal to the restatement's."""
    gc, gn, gh, gm = got
    rc, rn, rh, rm = ref.export_filtered()
    assert gc.shape == rc.shape, f"{what}: {gc.shape} vs {rc.shape}"
    assert np.array_equal(bits(gc), bits(rc)), f"{what}: centroids differ"
    assert np.array_equal(gn, rn), f"{what}: counts differ"
    assert np.array_equal(gh, rh), f"{what}: hits differ"
    assert np.array_equal(gm, rm), f"{what}: {int((gm != rm).sum())} voxels differ in misses"


def fresh_index(keys):
    """The occupancy index built from scratch from the stored keys -> (brick keys ascending, masks B x 8)."""
    v = dr.key_voxel(keys) + cr.HALF
    if v.shape[0] == 0:
        return np.zeros(0, np.uint64), np.zeros((0, 8), np.uint64)
    brick = ((v[:, 2] >> 3) << 36) | ((v[:, 1] >> 3) << 18) | (v[:, 0] >> 3)
    bit = ((v[:, 2] & 7) << 6) | ((v[:, 1] & 7) << 3) | (v[:, 0] & 7)
    ub, inv = np.unique(brick, return_inverse=True)
    masks = np.zeros((ub.size, 8), np.uint64)
    np.bitwise_or.at(masks, (inv, bit >> 6), np.left_shift(np.uint64(1), (bit & 63).astype(np.uint64)))
    return ub.astype(np.uint64), masks


def assert_index(c, ref, what):
    k, m = c.dense_carve_index()
    fk, fm = fresh_index(ref.keys)
    assert np.array_equal(k, fk) and np.array_equal(m, fm), f"{what}: the index is not a fresh build's"


@pytest.fixture(scope="module")
def runs(scene):
    from loam_velodyne_b200 import synth
    return {"vlp16": vr.moving_box_run(scene, synth.Lidar.vlp16(), 8),
            "hdl64": vr.moving_box_run(scene, synth.Lidar.hdl64(), 4)}


def test_edge_cases(build_libs):
    from loam_velodyne_b200 import api
    c = api.Ctx(0)
    try:
        c.dense_enable(cr.LEAF)
        for name, (stored, seen, origin, margin, mx, expect, _, repeat) in cr.edge_cases().items():
            c.dense_clear()
            c.dense_carving(0.0, 0.0)
            c.dense_carving(margin, mx)
            ref = cr.CarveMapRef(cr.LEAF, margin=margin, max_range=mx)
            c.cloud_upload(api.C_MAP_FULL, stored)
            c.dense_insert(api.C_MAP_FULL)
            ref.insert(stored)
            c.cloud_upload(api.C_MAP_FULL, seen)
            tw = np.array([0.0, 0.0, 0.0, *origin], np.float32)
            if name == "saturation":  # the restatement's case starts from SAT - 2; here 65537 passes from 0
                for _ in range(cr.SAT + 2):
                    c.dense_observe(api.C_MAP_FULL, tw)
                ref.misses = np.minimum(ref.misses + cr.SAT + 2, cr.SAT)
            else:
                for _ in range(repeat):
                    c.dense_observe(api.C_MAP_FULL, tw)
                    ref.observe(seen, tw)
            assert c.dense_export(evidence=True)[3].tolist() == expect, name
            assert_same(c.dense_export(evidence=True), ref, name)
    finally:
        c.close()


@pytest.mark.parametrize("lidar", ["vlp16", "hdl64"])
@pytest.mark.parametrize("leaf", [0.1, 0.2])
def test_observe_insert_sequences(build_libs, runs, lidar, leaf):
    """dense_observe + dense_insert at known poses from an empty map: the table and the index grow on the way; every
    field is checked after every sweep, and the index against a fresh build."""
    from loam_velodyne_b200 import api
    ref = cr.CarveMapRef(leaf, margin=0.5, max_range=60.0)
    c = api.Ctx(0)
    try:
        c.dense_enable(leaf)
        c.dense_carving(0.5, 60.0)
        slots = []
        for k, (pts, twist, _) in enumerate(runs[lidar]):
            pose = tilted(twist, k)
            c.cloud_upload(api.C_MAP_FULL, pts)
            c.dense_observe(api.C_MAP_FULL, pose)
            c.dense_insert(api.C_MAP_FULL)
            ref.sweep(pts, pose)
            assert_same(c.dense_export(evidence=True), ref, f"{lidar} leaf {leaf} sweep {k}")
            assert_index(c, ref, f"{lidar} leaf {leaf} sweep {k}")
            slots.append(c.dense_table_slots())
        assert slots[-1] > slots[0] and int(ref.misses.astype(bool).sum()) > 100
        print(f"{lidar} leaf {leaf}: {ref.keys.size} voxels, {int(ref.misses.astype(bool).sum())} with misses, "
              f"table slots {slots}")
    finally:
        c.close()


def test_small_table_growth_and_late_switch_on(build_libs, runs):
    """A cap that drops voxels, then growth mid-run; carve mode switched on with a map already stored builds its index
    from the table; clear and off drop it; inserts with the mode off still count hits and no misses."""
    from loam_velodyne_b200 import api
    pts = [r[0] for r in runs["vlp16"]]
    tw = [r[1] for r in runs["vlp16"]]
    c = api.Ctx(0)
    try:
        c.dense_enable(0.2, 5000)
        ref = cr.CarveMapRef(0.2, 5000, margin=1.0, max_range=80.0)
        for k in range(3):  # carve mode off: inserts only
            c.cloud_upload(api.C_MAP_FULL, pts[k])
            c.dense_insert(api.C_MAP_FULL)
            ref.insert(pts[k])
        assert c.dense_carve_index()[0].size == 0
        c.dense_enable(0.2)
        ref.max_voxels = 2**31 - 1
        c.dense_carving(1.0, 80.0)
        assert_index(c, ref, "switched on")
        for k in range(3, 8):
            c.cloud_upload(api.C_MAP_FULL, pts[k])
            c.dense_observe(api.C_MAP_FULL, tw[k])
            c.dense_insert(api.C_MAP_FULL)
            ref.sweep(pts[k], tw[k])
            assert_same(c.dense_export(evidence=True), ref, f"sweep {k}")
            assert_index(c, ref, f"sweep {k}")
        assert ref.stats()["dropped"] > 0 and c.dense_stats() == ref.stats()
        # new parameters keep the index
        c.dense_carving(2.0, 50.0)
        ref.set_carving(2.0, 50.0)
        c.cloud_upload(api.C_MAP_FULL, pts[0])
        c.dense_observe(api.C_MAP_FULL, tw[0])
        ref.observe(pts[0], tw[0])
        assert_same(c.dense_export(evidence=True), ref, "new parameters")
        # off: no index; inserts count hits, no misses
        c.dense_carving(0.0, 0.0)
        assert c.dense_carve_index()[0].size == 0
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_observe(api.C_MAP_FULL, tw[1])
        c.cloud_upload(api.C_MAP_FULL, pts[1])
        c.dense_insert(api.C_MAP_FULL)
        ref.insert(pts[1])
        assert_same(c.dense_export(evidence=True), ref, "off")
        # clear with the mode on: the index goes and restarts with the next insertion
        c.dense_carving(1.0, 80.0)
        ref.set_carving(1.0, 80.0)
        c.dense_clear()
        assert c.dense_carve_index()[0].size == 0
        ref = cr.CarveMapRef(0.2, margin=1.0, max_range=80.0)
        for k in (2, 3):
            c.cloud_upload(api.C_MAP_FULL, pts[k])
            c.dense_observe(api.C_MAP_FULL, tw[k])
            c.dense_insert(api.C_MAP_FULL)
            ref.sweep(pts[k], tw[k])
        assert_same(c.dense_export(evidence=True), ref, "after clear")
        assert_index(c, ref, "after clear")
    finally:
        c.close()


def test_modes_errors_and_launches(build_libs, runs):
    from loam_velodyne_b200 import api
    pts, tw = runs["vlp16"][0][0], runs["vlp16"][0][1]
    c = api.Ctx(0)
    try:
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_carving(1.0, 50.0)  # no dense map
        c.dense_enable(0.1)
        for bad in ((float("nan"), 50.0), (1.0, float("inf")), (-0.1, 50.0), (1.0, -1.0), (1.0, 65536 * 0.1 * 1.001)):
            with pytest.raises(api.LoamB200Error, match="invalid argument"):
                c.dense_carving(*bad)
        c.dense_carving(0.0, 65536 * 0.1)  # exactly the step bound
        with pytest.raises(api.LoamB200Error, match="invalid argument"):
            c.dense_enable(0.05)  # a leaf that would break the step bound of the carve mode on
        # the modes exclude each other; each may be turned off while the other is on
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_visibility(1.0, 2.0, 1.0)
        c.dense_visibility(0.0, 0.0, 0.0)
        c.dense_carving(0.0, 0.0)
        c.dense_visibility(1.0, 2.0, 1.0)
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_carving(1.0, 50.0)
        c.dense_carving(0.0, 0.0)
        c.dense_visibility(0.0, 0.0, 0.0)
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_observe(api.C_MAP_FULL, tw)  # both off
        # launches: with both modes off, an insertion launches what it launched before carve mode existed, and so
        # does one after carve mode was on and turned off; with it on, one more per insertion and 2 per observe
        c.cloud_upload(api.C_MAP_FULL, pts)

        def insert_launches():
            # the same cloud again and again: after two inserts neither the table nor the index grows any more
            # (dense_stats synchronises, so each insertion sizes from the stored voxels, not a running bound)
            for _ in range(2):
                c.dense_stats()
                c.dense_insert(api.C_MAP_FULL)
            c.dense_stats()
            before = c.launch_count()
            c.dense_insert(api.C_MAP_FULL)
            return c.launch_count() - before

        plain = insert_launches()
        c.dense_carving(1.0, 50.0)
        on = insert_launches()
        c.profile(True)
        before = c.launch_count()
        c.dense_observe(api.C_MAP_FULL, tw)
        assert c.launch_count() - before == 2
        prof = c.profile_get()
        assert sum(v[1] for k, v in prof.items() if k != "dense") == 0
        c.profile(False)
        c.dense_carving(0.0, 0.0)
        assert on == plain + 1 and insert_launches() == plain
        c.dense_clear()
    finally:
        c.close()
    s = api.Ctx(0)
    try:
        s.map_set_shard(0, 2)
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            s.dense_carving(1.0, 50.0)
    finally:
        s.close()


def mapping_run(scene, map_200k, carve):
    """The mapping stage as test_dense_visibility runs it, dense map on, carve mode on or off."""
    from loam_velodyne_b200 import api, synth
    reg = api.ScanRegistration()
    m = api.LaserMapping(0.1, 10)
    m.seed(*map_200k)
    m.enable_dense_map(0.1)
    if carve:
        m.enable_dense_carving()
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
    """The mapping stage's own run: every per-sweep output unchanged with carve mode on; its MAP_FULL clouds and poses
    through the restatement give the stage's evidence; the Ctx path on the same clouds gives the drop-in's."""
    from loam_velodyne_b200 import api
    off, _, _, m_off = mapping_run(scene, map_200k, False)
    on, fulls, poses, m = mapping_run(scene, map_200k, True)
    for i, (a, b) in enumerate(zip(off, on)):
        for x, y in zip(a, b):
            assert np.array_equal(bits(x), bits(y)), f"sweep {i}: an output changed with carve mode on"
    a, b = m_off.dense_map(), m.dense_map()
    assert np.array_equal(bits(a[0]), bits(b[0])) and np.array_equal(a[1], b[1])
    ref = cr.CarveMapRef(0.1)
    for pts, pose in zip(fulls, poses):
        ref.sweep(pts, pose)
    assert int(ref.misses.astype(bool).sum()) > 100
    got = m.dense_map(evidence=True)
    assert_same(got, ref, "mapping stage")
    c = api.Ctx(0)
    try:
        c.dense_enable(0.1)
        c.dense_carving()
        for pts, pose in zip(fulls, poses):
            c.cloud_upload(api.C_MAP_FULL, pts)
            c.dense_observe(api.C_MAP_FULL, pose)
            c.dense_insert(api.C_MAP_FULL)
        ctx = c.dense_export(evidence=True)
        assert np.array_equal(bits(ctx[0]), bits(got[0])) and all(np.array_equal(x, y) for x, y in zip(ctx[1:], got[1:]))
    finally:
        c.close()
    assert m.dense_map(1.0)[0].shape[0] < a[0].shape[0]


def test_pipeline_in_flight(build_libs, scene):
    from loam_velodyne_b200 import api, synth
    lidar = synth.Lidar.vlp16()
    sweeps = [synth.make_sweep(scene, lidar, i, yaw_rate=math.radians(5.0)) for i in range(3)]
    pl = api.Pipeline()
    pl.mapping.enable_dense_map(0.1)
    pl.mapping.enable_dense_carving()
    for q, rs in sweeps:
        pl.submit(q, rs)
    with pytest.raises(api.LoamB200Error, match="in flight"):
        pl.mapping.enable_dense_carving(0.0, 0.0)
    while pl.collect(wait=True) is not None:
        pass
    _, _, hits, misses = pl.mapping.dense_map(evidence=True)
    assert hits.size > 10000 and int(misses.astype(bool).sum()) > 0
    pl.mapping.enable_dense_carving(0.0, 0.0)
