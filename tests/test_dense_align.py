"""Alignment against the whole-run voxel map on the GPU (csrc/densemap.cuh: dense_align_kernel; loam_b200_dense_align)
against the numpy restatement (tests/align_reference.py): each iteration bit for bit (matches, coefficients, selected
flags and the normal equations, NaN equal to NaN), the loop against a replay through the iteration entry point, pose
recovery, snapshot and round-trip semantics, the error paths, and the mapping stage's own map."""
import math

import numpy as np
import pytest

import align_reference as ar
import dense_reference as dr
from test_align_reference import BAR_DEG, BAR_M, HELD_OUT, MAP_TWISTS, coarse_to_fine, lidars

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def drv(build_libs):
    from oracle import pydriver
    return pydriver.best()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def ne_bits(ne, ss):
    return np.concatenate([bits(ne["AtA"]).ravel(), bits(ne["AtB"]), [ne["n_selected"], ne["n_corner_selected"]],
                           bits(np.float32(ss)).ravel()])


def ref_ne_bits(r):
    AtA, AtB, n_sel, ss = ar.normal_eq(r)
    return np.concatenate([bits(AtA).ravel(), bits(AtB), [n_sel, 0], bits(np.float32(ss)).ravel()])


def assert_iterate(c, tgt, pts, twist, radius, what):
    ne, ss, match, coeff, sel = c.dense_align_iterate(pts, twist, radius, debug=True)
    r, rm, rc, rs = ar.iterate(tgt, pts, twist, radius)
    assert np.array_equal(match, rm), f"{what}: {int((match != rm).sum())} matches differ"
    assert np.array_equal(bits(coeff), bits(rc)), f"{what}: coefficients differ"
    assert np.array_equal(sel.astype(bool), rs), f"{what}: selected flags differ"
    assert np.array_equal(ne_bits(ne, ss), ref_ne_bits(r)), f"{what}: normal equations differ"
    again = c.dense_align_iterate(pts, twist, radius)
    assert np.array_equal(ne_bits(*again), ne_bits(ne, ss)), f"{what}: a second call differs"
    return ne


def map_ctx(scene, lidar, leaf):
    """A context with the whole-run map of the static map sweeps, and the same map in the restatement."""
    from loam_velodyne_b200 import api
    c = api.Ctx(0)
    c.dense_enable(leaf)
    ref = dr.DenseMapRef(leaf)
    for k, tw in enumerate(MAP_TWISTS):
        w = ar.static_sweep(scene, lidar, tw, seed=k)[1]
        c.cloud_upload(api.C_MAP_FULL, w)
        c.dense_insert(api.C_MAP_FULL)
        ref.insert(w)
    return c, ref


@pytest.mark.parametrize("leaf", [0.1, 0.2, 0.4])
def test_iterate_hdl64(build_libs, scene, drv, leaf):
    """Targets built on the GPU from HDL-64E sweeps at three leaves; a held-out sweep at search radius 1, 2 and 3, at
    the zero pose and at rotated poses near the truth."""
    from loam_velodyne_b200 import synth
    lidar = synth.Lidar.hdl64(1024)
    c, ref = map_ctx(scene, lidar, leaf)
    try:
        vp = (0.5, 1.0, -2.0)
        n = c.dense_target_build(None, 2, vp)
        tgt = ar.built_target(ref, 2, vp, drv)
        assert n == tgt.keys.size
        pts = ar.static_sweep(scene, lidar, HELD_OUT[1].astype(np.float64), seed=60)[0]
        pts[::501, 1] = np.nan
        rotated = HELD_OUT[1] + np.array([0.02, -0.03, 0.01, 0.1, 0.05, -0.2], np.float32)
        for radius in (1, 2, 3):
            for twist in (np.zeros(6, np.float32), HELD_OUT[1], rotated):
                ne = assert_iterate(c, tgt, pts, twist, radius, f"leaf {leaf} radius {radius} twist {twist}")
                if twist is not HELD_OUT[1]:
                    continue
                assert ne["n_selected"] > pts.shape[0] // 10
    finally:
        c.close()


@pytest.mark.parametrize("name", list(ar.edge_cases()))
def test_edge_cases(build_libs, name):
    """The hand-made cases, loaded into a context without the map."""
    from loam_velodyne_b200 import api
    cent, nrm, pts, twist, radius, _ = ar.edge_cases()[name]
    tgt = ar.loaded_target(ar.EDGE_LEAF, cent, nrm)
    c = api.Ctx(0)
    try:
        c.dense_target_load(ar.EDGE_LEAF, cent, nrm)
        for r in sorted({radius, 1, 3}):
            assert_iterate(c, tgt, pts, twist, r, f"{name} radius {r}")
    finally:
        c.close()


def replay(c, pts, twist, radius, max_iterations, drv=None):
    """The loop of align_reference with each iteration's sums from the GPU's iteration entry point."""
    def step(t):
        ne, ss = c.dense_align_iterate(pts, t, radius)
        r = np.zeros(32, np.float32)
        k = 0
        for i in range(6):
            for j in range(i, 6):
                r[k] = ne["AtA"][i, j]
                k += 1
        r[21:27] = ne["AtB"]
        r[27] = np.float32(ne["n_selected"])
        r[28] = ss
        return r
    return ar.align(ar.Target(1.0, [0], np.zeros((1, 4)), np.zeros((1, 4))), pts, twist, radius, max_iterations,
                    step=step, drv=drv)


def test_align_equals_replay(build_libs, scene, drv):
    """dense_align is the replay bit for bit on recovery runs, also coarse to fine; on the one-plane target it reports
    degenerate and matches a replay with the first solve's projection within 2e-4."""
    from loam_velodyne_b200 import api
    lidar = lidars()["vlp16"]
    c, _ = map_ctx(scene, lidar, 0.2)
    try:
        c.dense_target_build(None, 2)
        exact = 0
        for h in range(3):
            pts = ar.static_sweep(scene, lidar, HELD_OUT[h].astype(np.float64), seed=100 + h)[0]
            init = (HELD_OUT[h] + ar.perturbations(h, 1)[0]).astype(np.float32)
            for radius, it in ((3, 30), (1, 30), (2, 3)):
                got, info = c.dense_align(pts, init, radius, it)
                want, winfo = replay(c, pts, init, radius, it, drv=drv)
                assert info["degenerate"] == winfo["degenerate"], (h, radius, info, winfo)
                if info["degenerate"]:  # the projection of the replay is the checker's, in float64
                    np.testing.assert_allclose(got, want, rtol=0, atol=2e-4)
                    continue
                assert np.array_equal(bits(got), bits(want)) and info == winfo, (h, radius, info, winfo)
                exact += 1
        assert exact >= 3
    finally:
        c.close()
    cent, nrm, pts = ar.plane_case()
    c = api.Ctx(0)
    try:
        c.dense_target_load(ar.EDGE_LEAF, cent, nrm)
        init = np.array([0.01, 0.0, -0.01, 0.0, 0.05, 0.0], np.float32)
        got, info = c.dense_align(pts, init, 1, 10)
        want, winfo = replay(c, pts, init, 1, 10, drv=drv)
        assert info["degenerate"] and winfo["degenerate"] and info["iterations"] == winfo["iterations"]
        np.testing.assert_allclose(got, want, rtol=0, atol=2e-4)
    finally:
        c.close()


@pytest.mark.parametrize("leaf", [0.1, 0.2])
@pytest.mark.parametrize("sensor", ["vlp16", "hdl64"])
def test_pose_recovery(build_libs, scene, drv, sensor, leaf):
    """Every held-out sweep from two ~0.3 m / 2 deg perturbations, radius 3 then 1, within the restatement's bars."""
    lidar = lidars()[sensor]
    c, _ = map_ctx(scene, lidar, leaf)
    try:
        c.dense_target_build(None, 2)
        for h in range(3):
            truth = HELD_OUT[h]
            pts = ar.static_sweep(scene, lidar, truth.astype(np.float64), seed=100 + h)[0]
            for pert in ar.perturbations(h, 2):
                got, info = coarse_to_fine(c.dense_align, pts, (truth + pert).astype(np.float32))
                e_m, e_deg = ar.twist_error(got, truth)
                assert info["converged"] and e_m <= BAR_M and e_deg <= BAR_DEG, (sensor, leaf, h, e_m, e_deg, info)
    finally:
        c.close()


def test_snapshot_and_round_trip(build_libs, scene):
    """An insert after the build leaves the results as they were, a rebuild changes them; export -> load into a fresh
    context with the map off gives the same bits; a duplicate voxel in a load is refused."""
    from loam_velodyne_b200 import api, synth
    lidar = lidars()["vlp16"]
    c, _ = map_ctx(scene, lidar, 0.1)
    try:
        vp = (0.0, 0.0, 0.0)
        c.dense_target_build(1.0, 2, vp)
        pts = ar.static_sweep(scene, lidar, HELD_OUT[0].astype(np.float64), seed=100)[0]
        init = (HELD_OUT[0] + ar.perturbations(0, 1)[0]).astype(np.float32)
        first = c.dense_align(pts, init, 3, 10)
        it1 = c.dense_align_iterate(pts, init, 2)
        cent, _, nrm = c.dense_export_normals(1.0, 2, vp)
        extra = ar.static_sweep(scene, synth.Lidar.hdl64(512), HELD_OUT[0].astype(np.float64), seed=7)[1]
        c.cloud_upload(api.C_MAP_FULL, extra)
        c.dense_insert(api.C_MAP_FULL)
        after = c.dense_align(pts, init, 3, 10)
        assert np.array_equal(bits(after[0]), bits(first[0])) and after[1] == first[1]
        assert np.array_equal(ne_bits(*c.dense_align_iterate(pts, init, 2)), ne_bits(*it1))
        c.dense_target_build(1.0, 2, vp)
        assert not np.array_equal(ne_bits(*c.dense_align_iterate(pts, init, 2)), ne_bits(*it1))
    finally:
        c.close()
    f = api.Ctx(0)
    try:
        f.dense_target_load(0.1, cent[::-1], nrm[::-1])
        got = f.dense_align(pts, init, 3, 10)
        assert np.array_equal(bits(got[0]), bits(first[0])) and got[1] == first[1]
        assert np.array_equal(ne_bits(*f.dense_align_iterate(pts, init, 2)), ne_bits(*it1))
        dup = np.concatenate([cent, cent[3:4] + np.float32(1e-3)])
        with pytest.raises(api.LoamB200Error, match="invalid argument"):
            f.dense_target_load(0.1, dup, np.concatenate([nrm, nrm[3:4]]))
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):  # a failed load leaves no target
            f.dense_align(pts, init, 1, 5)
    finally:
        f.close()


def test_errors(build_libs, scene):
    import ctypes as C
    from loam_velodyne_b200 import api
    pts = np.ones((100, 4), np.float32)
    c = api.Ctx(0)
    try:
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_align(pts, np.zeros(6), 1, 5)  # no target
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_align_iterate(pts, np.zeros(6), 1)
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_target_build()  # map off
        for leaf, cent in ((0.0, pts), (float("nan"), pts), (-1.0, pts), (0.1, np.full((2, 4), np.inf, np.float32)),
                           (0.1, np.array([[3e6, 0, 0, 0]], np.float32))):
            with pytest.raises(api.LoamB200Error, match="invalid argument"):
                c.dense_target_load(leaf, cent, np.zeros_like(cent))
        c.dense_target_load(0.5, np.zeros((0, 4), np.float32), np.zeros((0, 4), np.float32))
        got, info = c.dense_align(pts, np.array([0.1, 0.2, 0.3, 1, 2, 3], np.float32), 1, 5)  # empty target
        assert np.array_equal(got, np.array([0.1, 0.2, 0.3, 1, 2, 3], np.float32)) and not info["converged"]
        cent, nrm, _ = ar.plane_case()
        c.dense_target_load(ar.EDGE_LEAF, cent, nrm)
        got, info = c.dense_align(pts[:0], np.zeros(6), 1, 5)  # empty cloud
        assert info["iterations"] == 0 and not info["converged"]
        for radius, iters, tw in ((0, 5, np.zeros(6)), (4, 5, np.zeros(6)), (1, 0, np.zeros(6)), (1, 101, np.zeros(6)),
                                  (1, 5, np.array([np.nan, 0, 0, 0, 0, 0])), (1, 5, np.array([0, 0, 0, 0, np.inf, 0]))):
            with pytest.raises(api.LoamB200Error, match="invalid argument"):
                c.dense_align(pts, tw, radius, iters)
        L = c.L
        ne = api.NormalEq()
        p = api.make_pose(np.zeros(6))
        r = api.AlignResult()
        assert L.loam_b200_dense_align_iterate(c.h, api._fp(pts), 100, 0, C.byref(p), 1, None, None, None, None,
                                               None) == -1
        assert L.loam_b200_dense_align_iterate(c.h, None, 100, 0, C.byref(p), 1, C.byref(ne), None, None, None,
                                               None) == -1
        assert L.loam_b200_dense_align(c.h, api._fp(pts), 100, 0, None, 1, 5, C.byref(r)) == -1
        assert L.loam_b200_dense_align(c.h, api._fp(pts), 100, 0, C.byref(p), 1, 5, None) == -1
        assert L.loam_b200_dense_target_build(c.h, math.inf, 1, None, None) == -1
    finally:
        c.close()
    s = api.Ctx(0)
    try:
        s.dense_enable(0.2)
        s.map_set_shard(0, 2)
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            s.dense_target_build()
    finally:
        s.close()
    from loam_velodyne_b200 import synth
    lidar = synth.Lidar.vlp16()
    sweeps = [synth.make_sweep(scene, lidar, i, yaw_rate=math.radians(5.0)) for i in range(3)]
    pl = api.Pipeline()
    pl.mapping.enable_dense_map(0.1)
    for q, rs in sweeps:
        pl.submit(q, rs)
    for call in (lambda: pl.mapping.build_dense_target(), lambda: pl.mapping.load_dense_target(0.5, cent, nrm),
                 lambda: pl.mapping.align_to_dense_target(pts, np.zeros(6))):
        with pytest.raises(api.LoamB200Error, match="in flight"):
            call()
    while pl.collect(wait=True) is not None:
        pass
    assert pl.mapping.build_dense_target() > 0
    pl.sync()


SUMS = [(0.0, 0.05 * i, 0.0, 0.4 * i, 0.02 * i, 0.9 * i) for i in range(12)]


def test_mapping_stage(build_libs, scene, map_200k):
    """VLP-16 through the mapping stage with the dense map on: sweep k's sensor-frame full cloud aligned from a perturbed
    transformAftMapped returns to it; the drop-in path equals the Ctx path (target loaded from the export) bit for bit."""
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
    c = api.Ctx(0)
    try:
        c.dense_target_load(0.1, cent, nrm)
        for k in (3, 8):
            init = (afts[k] + ar.perturbations(k, 1, metres=0.3, degrees=2.0)[0]).astype(np.float32)
            got, info = coarse_to_fine(m.align_to_dense_target, clouds[k], init)
            want, winfo = coarse_to_fine(c.dense_align, clouds[k], init)
            assert np.array_equal(bits(got), bits(want)) and info == winfo, (info, winfo)
            e_m, e_deg = ar.twist_error(got, afts[k])
            assert info["converged"] and e_m <= BAR_M and e_deg <= BAR_DEG, (k, e_m, e_deg, info)
    finally:
        c.close()
