"""Relocalisation against the whole-run voxel map on the GPU (csrc/densemap.cuh: dense_align_kernel over a hypothesis
list; loam_b200_dense_score / _align_batch / _relocalize): the score equals the iteration entry point bit for bit at
every pose (also across the 65 535-pose chunk boundary), the batch equals one dense_align per pose, relocalize equals
a replay of the restated rules (tests/reloc_reference.py) over score and batch, recovery from an unknown heading and a
prior 1.5 m off, the mapping stage's drop-in path, and the error paths.  96 s together with test_dense_align.py on an
H100 80GB HBM3 at 700 W."""
import math

import numpy as np
import pytest

import align_reference as ar
import reloc_reference as rr
from test_align_reference import BAR_DEG, BAR_M, HELD_OUT, lidars
from test_dense_align import map_ctx

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def assert_score(c, pts, twists, radius, what):
    sel, ss = c.dense_score(pts, twists, radius)
    for h, t in enumerate(twists):
        ne, s = c.dense_align_iterate(pts, t, radius)
        assert sel[h] == ne["n_selected"] and bits(ss[h]) == bits(s), (what, h, sel[h], ne["n_selected"], ss[h], s)
    return sel


def near_twists(truth, n, seed, metres=1.0, degrees=10.0):
    rng = np.random.RandomState(seed)
    out = [truth]
    for _ in range(n - 1):
        d = np.concatenate([rng.uniform(-1, 1, 3) * math.radians(degrees) * np.array([0.1, 1.0, 0.1]),
                            rng.uniform(-1, 1, 3) * metres * np.array([1.0, 0.1, 1.0])])
        out.append(truth + d)
    return np.array(out, np.float32)


@pytest.mark.parametrize("leaf", [0.1, 0.2, 0.4])
def test_score_hdl64(build_libs, scene, leaf):
    from loam_velodyne_b200 import synth
    lidar = synth.Lidar.hdl64(1024)
    c, _ = map_ctx(scene, lidar, leaf)
    try:
        c.dense_target_build(None, 2, (0.5, 1.0, -2.0))
        pts = ar.static_sweep(scene, lidar, HELD_OUT[1].astype(np.float64), seed=60)[0]
        pts[::501, 1] = np.nan
        tw = near_twists(HELD_OUT[1], 6, seed=int(leaf * 10))
        for radius in (1, 2, 3):
            sel = assert_score(c, pts, tw, radius, f"leaf {leaf} radius {radius}")
            assert sel[0] > pts.shape[0] // 10
    finally:
        c.close()


def test_score_edge_cases_and_chunks(build_libs):
    from loam_velodyne_b200 import api
    for name, (cent, nrm, pts, twist, radius, _) in ar.edge_cases().items():
        c = api.Ctx(0)
        try:
            c.dense_target_load(ar.EDGE_LEAF, cent, nrm)
            tw = np.array([twist, twist + np.float32(0.01), twist], np.float32)
            for r in sorted({radius, 1, 3}):
                assert_score(c, pts, tw, r, f"{name} radius {r}")
        finally:
            c.close()
    # 70 000 poses of a few-hundred-point cloud: two launches (65 535 + 4 465); every pose against the iteration entry point
    cent, nrm, pts = ar.plane_case(n=300)
    c = api.Ctx(0)
    try:
        c.dense_target_load(ar.EDGE_LEAF, cent, nrm)
        k = 70_000
        tw = np.zeros((k, 6), np.float32)
        tw[:, 4] = np.linspace(-0.3, 0.3, k, dtype=np.float32)
        tw[:, 0] = np.linspace(-0.05, 0.05, k, dtype=np.float32)
        sel, ss = c.dense_score(pts, tw, 1)
        want_sel, want_ss = np.zeros(k, np.int32), np.zeros(k, np.float32)
        for h in range(k):
            ne, want_ss[h] = c.dense_align_iterate(pts, tw[h], 1)
            want_sel[h] = ne["n_selected"]
        assert np.array_equal(sel, want_sel), np.nonzero(sel != want_sel)[0][:10]
        assert np.array_equal(bits(ss), bits(want_ss)), np.nonzero(bits(ss) != bits(want_ss))[0][:10]
        assert (sel > 0).all()
        sel2, ss2 = c.dense_score(pts, tw[65_530:65_540], 1)  # another chunking of the same poses
        assert np.array_equal(sel2, sel[65_530:65_540]) and np.array_equal(bits(ss2), bits(ss[65_530:65_540]))
    finally:
        c.close()


def assert_batch(c, pts, tw, radius, it):
    got, infos = c.dense_align_batch(pts, tw, radius, it)
    for h, t in enumerate(tw):
        want, winfo = c.dense_align(pts, t, radius, it)
        assert np.array_equal(bits(got[h]), bits(want)) and infos[h] == winfo, (h, infos[h], winfo)
    return got, infos


def test_align_batch(build_libs, scene):
    from loam_velodyne_b200 import api
    lidar = lidars()["vlp16"]
    c, _ = map_ctx(scene, lidar, 0.2)
    try:
        c.dense_target_build(None, 2)
        pts = ar.static_sweep(scene, lidar, HELD_OUT[1].astype(np.float64), seed=101)[0]
        tw = near_twists(HELD_OUT[1], 7, seed=3, metres=0.6, degrees=6.0)
        tw = np.concatenate([tw, tw[2:4]])  # duplicates
        for radius, it in ((1, 30), (2, 3)):
            assert_batch(c, pts, tw, radius, it)
        _, infos = assert_batch(c, pts, tw, 3, 30)
        assert len({i["iterations"] for i in infos}) > 1  # the runs stop at different iterations
    finally:
        c.close()
    cent, nrm, pts = ar.plane_case()
    c = api.Ctx(0)
    try:
        c.dense_target_load(ar.EDGE_LEAF, cent, nrm)
        tw = np.array([[0.01, 0.0, -0.01, 0.0, 0.05, 0.0], [0.0, 0.0, 0.02, 0.1, -0.05, 0.0]], np.float32)
        _, infos = assert_batch(c, pts, tw, 1, 10)
        assert all(i["degenerate"] for i in infos)
        got, infos = c.dense_align_batch(pts[:0], tw, 1, 10)  # empty cloud
        assert np.array_equal(got, tw) and all(i["iterations"] == 0 for i in infos)
        assert (c.dense_score(pts[:0], tw, 1)[0] == 0).all()
        c.dense_target_load(0.5, np.zeros((0, 4), np.float32), np.zeros((0, 4), np.float32))  # empty target
        got, infos = c.dense_align_batch(pts, tw, 1, 10)
        assert np.array_equal(got, tw) and all(i["iterations"] == 0 for i in infos)
        assert c.dense_relocalize(pts, tw) == []
    finally:
        c.close()


def same_candidates(a, b):
    assert len(a) == len(b), (len(a), len(b))
    for x, y in zip(a, b):
        for key in ("hypothesis", "score_selected", "selected"):
            assert x[key] == y[key], (key, x, y)
        assert bits(x["rms"]) == bits(y["rms"])
        for stage in ("coarse", "fine"):
            assert np.array_equal(bits(x[stage][0]), bits(y[stage][0])) and x[stage][1] == y[stage][1], stage


def gpu_replay(c, pts, hyps, prm, cap):
    return rr.relocalize(lambda t, r: c.dense_score(pts, t, r),
                         lambda t, r, it: c.dense_align_batch(pts, t, r, it), hyps, prm, cap)


def test_relocalize_equals_replay(build_libs, scene):
    from loam_velodyne_b200 import api
    lidar = lidars()["hdl64"]
    c, _ = map_ctx(scene, lidar, 0.2)
    try:
        c.dense_target_build(None, 2)
        truth = HELD_OUT[2]
        pts = ar.static_sweep(scene, lidar, truth.astype(np.float64), seed=102)[0]
        hyps = api.reloc_grid(truth + np.array([0, 0.3, 0, 0.4, 0, -0.3], np.float32), 15.0, None, 1.0, 1)
        for prm in (api.RelocParams.default(), api.RelocParams(2, 3, 1, 5, 8, 2.0, 30.0),
                    api.RelocParams(3, 2, 2, 40, 5, 0.0, 0.0)):
            got = c.dense_relocalize(pts, hyps, prm, cap=8)
            same_candidates(got, gpu_replay(c, pts, hyps, prm, 8))
            assert got
    finally:
        c.close()


@pytest.mark.parametrize("leaf", [0.1, 0.2])
@pytest.mark.parametrize("sensor", ["vlp16", "hdl64"])
def test_basin_contains_grid_corner(build_libs, scene, sensor, leaf):
    """From the recommended grid's worst-case corner (half a yaw step and half an x-z step on both ground axes) in 4
    diagonal directions with both yaw signs, every held-out sweep aligns coarse to fine within the bars."""
    from loam_velodyne_b200 import api
    lidar = lidars()[sensor]
    c, _ = map_ctx(scene, lidar, leaf)
    dyaw, dxz = math.radians(api.RELOC_YAW_STEP_DEG / 2.0), api.RELOC_XZ_STEP / 2.0
    try:
        c.dense_target_build(None, 2)
        for h in range(3):
            truth = HELD_OUT[h]
            pts = ar.static_sweep(scene, lidar, truth.astype(np.float64), seed=100 + h)[0]
            init = np.array([truth + np.array([0, sy * dyaw, 0, sx * dxz, 0, sz * dxz], np.float32)
                             for sy in (1, -1) for sx in (1, -1) for sz in (1, -1)], np.float32)
            coarse, _ = c.dense_align_batch(pts, init, 3, 30)
            fine, infos = c.dense_align_batch(pts, coarse, 1, 30)
            for j in range(init.shape[0]):
                e_m, e_deg = ar.twist_error(fine[j], truth)
                assert infos[j]["converged"] and e_m <= BAR_M and e_deg <= BAR_DEG, (sensor, leaf, h, j, e_m, e_deg)
    finally:
        c.close()


@pytest.mark.parametrize("leaf", [0.1, 0.2])
@pytest.mark.parametrize("sensor", ["vlp16", "hdl64"])
def test_recovery(build_libs, scene, sensor, leaf):
    """Every held-out sweep from an unknown heading (full circle at the recommended step) and a prior 1.5 m off in a
    random direction on the ground plane: candidate 0 is within the alignment bars of the truth."""
    from loam_velodyne_b200 import api
    lidar = lidars()[sensor]
    c, _ = map_ctx(scene, lidar, leaf)
    rng = np.random.RandomState(7)
    try:
        c.dense_target_build(None, 2)
        for h in range(3):
            truth = HELD_OUT[h]
            pts = ar.static_sweep(scene, lidar, truth.astype(np.float64), seed=100 + h)[0]
            a = rng.uniform(0, 2 * math.pi)
            prior = truth + np.array([0, rng.uniform(-math.pi, math.pi), 0, 1.5 * math.cos(a), 0, 1.5 * math.sin(a)],
                                     np.float32)
            hyps = api.reloc_grid(prior, api.RELOC_YAW_STEP_DEG, None, api.RELOC_XZ_STEP, api.RELOC_XZ_STEPS)
            cands = c.dense_relocalize(pts, hyps)
            assert cands, (sensor, leaf, h)
            e_m, e_deg = ar.twist_error(cands[0]["fine"][0], truth)
            gap = cands[0]["selected"] - (cands[1]["selected"] if len(cands) > 1 else 0)
            print(f"{sensor} leaf {leaf} sweep {h}: {e_m * 1000:.1f} mm {e_deg:.3f} deg, {len(cands)} candidates, "
                  f"selected {cands[0]['selected']} gap {gap}")
            assert e_m <= BAR_M and e_deg <= BAR_DEG, (sensor, leaf, h, e_m, e_deg, cands[0])
    finally:
        c.close()


def test_mapping_stage(build_libs, scene, map_200k):
    """On the mapping stage's own map: relocalise a sweep from transformAftMapped turned by 90 deg and moved by 1 m; the
    drop-in path equals the Ctx path (target loaded from the export) bit for bit."""
    from loam_velodyne_b200 import api, synth
    from test_dense_align import SUMS
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
    m.build_dense_target(None, 2, vp)
    cent, _, nrm = m.dense_map_normals(None, 2, vp)
    c = api.Ctx(0)
    try:
        c.dense_target_load(0.1, cent, nrm)
        k = 8
        prior = (afts[k] + np.array([0, math.pi / 2, 0, 0.6, 0, 0.8], np.float32)).astype(np.float32)
        hyps = api.reloc_grid(prior, api.RELOC_YAW_STEP_DEG, None, api.RELOC_XZ_STEP, api.RELOC_XZ_STEPS)
        got = m.relocalize_in_dense_target(clouds[k], hyps)
        same_candidates(got, c.dense_relocalize(clouds[k], hyps))
        e_m, e_deg = ar.twist_error(got[0]["fine"][0], afts[k])
        assert e_m <= BAR_M and e_deg <= BAR_DEG, (e_m, e_deg, got[0])
        sel, ss = m.score_dense_target(clouds[k], hyps[:50], 3)
        sel2, ss2 = c.dense_score(clouds[k], hyps[:50], 3)
        assert np.array_equal(sel, sel2) and np.array_equal(bits(ss), bits(ss2))
        t1, i1 = m.align_to_dense_target_batch(clouds[k], hyps[:5], 3, 10)
        t2, i2 = c.dense_align_batch(clouds[k], hyps[:5], 3, 10)
        assert np.array_equal(bits(t1), bits(t2)) and i1 == i2
    finally:
        c.close()


def test_errors(build_libs, scene):
    import ctypes as C
    from loam_velodyne_b200 import api
    pts = np.ones((100, 4), np.float32)
    tw = np.zeros((2, 6), np.float32)
    c = api.Ctx(0)
    try:
        for call in (lambda: c.dense_score(pts, tw, 1), lambda: c.dense_align_batch(pts, tw, 1, 5),
                     lambda: c.dense_relocalize(pts, tw)):
            with pytest.raises(api.LoamB200Error, match="invalid call sequence"):  # no target
                call()
        cent, nrm, _ = ar.plane_case()
        c.dense_target_load(ar.EDGE_LEAF, cent, nrm)
        bad_tw = tw.copy()
        bad_tw[1, 3] = np.inf
        for call in (lambda: c.dense_score(pts, tw, 0), lambda: c.dense_score(pts, tw, 4),
                     lambda: c.dense_score(pts, tw[:0], 1), lambda: c.dense_score(pts, bad_tw, 1),
                     lambda: c.dense_align_batch(pts, tw, 1, 0), lambda: c.dense_align_batch(pts, tw, 1, 101),
                     lambda: c.dense_align_batch(pts, bad_tw, 1, 5), lambda: c.dense_align_batch(pts, tw[:0], 1, 5),
                     lambda: c.dense_relocalize(pts, tw, api.RelocParams(3, 3, 1, 0, 30, 0.5, 5.0)),
                     lambda: c.dense_relocalize(pts, tw, api.RelocParams(3, 3, 1, 1025, 30, 0.5, 5.0)),
                     lambda: c.dense_relocalize(pts, tw, api.RelocParams(0, 3, 1, 4, 30, 0.5, 5.0)),
                     lambda: c.dense_relocalize(pts, tw, api.RelocParams(3, 4, 1, 4, 30, 0.5, 5.0)),
                     lambda: c.dense_relocalize(pts, tw, api.RelocParams(3, 3, 0, 4, 30, 0.5, 5.0)),
                     lambda: c.dense_relocalize(pts, tw, api.RelocParams(3, 3, 1, 4, 0, 0.5, 5.0)),
                     lambda: c.dense_relocalize(pts, tw, api.RelocParams(3, 3, 1, 4, 30, -0.5, 5.0)),
                     lambda: c.dense_relocalize(pts, tw, api.RelocParams(3, 3, 1, 4, 30, 0.5, -1.0)),
                     lambda: c.dense_relocalize(pts, tw, api.RelocParams(3, 3, 1, 4, 30, math.nan, 5.0)),
                     lambda: c.dense_relocalize(pts, bad_tw), lambda: c.dense_relocalize(pts, tw, cap=0)):
            with pytest.raises(api.LoamB200Error, match="invalid argument"):
                call()
        L = c.L
        p = (api.Pose * 2)(api.make_pose(tw[0]), api.make_pose(tw[1]))
        sel = np.zeros(2, np.int32)
        ss = np.zeros(2, np.float32)
        assert L.loam_b200_dense_score(c.h, api._fp(pts), 100, 0, None, 2, 1, api._ip(sel), api._fp(ss)) == -1
        assert L.loam_b200_dense_score(c.h, api._fp(pts), 100, 0, p, 2, 1, None, api._fp(ss)) == -1
        assert L.loam_b200_dense_score(c.h, api._fp(pts), 100, 0, p, (1 << 20) + 1, 1, api._ip(sel), api._fp(ss)) == -1
        assert L.loam_b200_dense_align_batch(c.h, api._fp(pts), 100, 0, p, 2, 1, 5, None) == -1
        prm = api.RelocParams.default()
        n = C.c_int(0)
        assert L.loam_b200_dense_relocalize(c.h, api._fp(pts), 100, 0, p, 2, None, None, 4, C.byref(n)) == -1
        assert c.dense_relocalize(pts, tw, prm) == []  # nothing reaches 50 selected: no candidate, no error
    finally:
        c.close()
    # the grid (host only)
    with pytest.raises(api.LoamB200Error, match="invalid argument"):
        api.reloc_grid(np.zeros(6), 0.0, 3, 1.0, 1)
    with pytest.raises(api.LoamB200Error, match="invalid argument"):
        api.reloc_grid(np.zeros(6), 5.0, 3, -1.0, 1)
    with pytest.raises(api.LoamB200Error, match="invalid argument"):
        api.reloc_grid(np.zeros(6), 5.0, -1, 1.0, 1)
    with pytest.raises(api.LoamB200Error, match="invalid argument"):
        api.reloc_grid(np.zeros(6), 1.0, 180, 0.1, 100)  # more than 1 << 20 poses
    # in-flight refusal on a pipeline
    from loam_velodyne_b200 import synth
    lidar = synth.Lidar.vlp16()
    sweeps = [synth.make_sweep(scene, lidar, i, yaw_rate=math.radians(5.0)) for i in range(3)]
    pl = api.Pipeline()
    pl.mapping.enable_dense_map(0.1)
    for q, rs in sweeps:
        pl.submit(q, rs)
    for call in (lambda: pl.mapping.score_dense_target(pts, tw), lambda: pl.mapping.align_to_dense_target_batch(pts, tw),
                 lambda: pl.mapping.relocalize_in_dense_target(pts, tw)):
        with pytest.raises(api.LoamB200Error, match="in flight"):
            call()
    while pl.collect(wait=True) is not None:
        pass
    pl.sync()
