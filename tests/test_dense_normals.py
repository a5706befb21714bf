"""Normals of the whole-run voxel map's export on the GPU (csrc/densemap.cuh: dense_normals_kernel) against the numpy
restatement (tests/normals_reference.py), bit for bit with no tolerance: normals and curvature as float bits, NaN in
the same places, and centroids and counts equal to dense_export(_filtered) at the same ratio."""
import math

import numpy as np
import pytest

import dense_reference as dr
import normals_reference as nr

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_CAPACITY = -1, -5


@pytest.fixture(scope="module")
def drv(build_libs):
    from oracle import pydriver
    return pydriver.best()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def registered(pts, yaw, t):
    c, s = np.float32(math.cos(yaw)), np.float32(math.sin(yaw))
    p = np.array(pts, np.float32, copy=True)
    x, z = p[:, 0].copy(), p[:, 2].copy()
    p[:, 0] = c * x + s * z + np.float32(t[0])
    p[:, 1] = p[:, 1] + np.float32(t[1])
    p[:, 2] = -s * x + c * z + np.float32(t[2])
    return p


def box_cloud(n, lo, hi, seed, leaf):
    """n points in a box, snapped so that many share a voxel."""
    rng = np.random.RandomState(seed)
    p = rng.uniform(lo, hi, (n, 3)).astype(np.float32)
    p = (np.round(p / (leaf * 0.25)) * (leaf * 0.25) + rng.uniform(-1e-3, 1e-3, (n, 3))).astype(np.float32)
    inten = (rng.uniform(0, 1, n) * 10.0 ** rng.randint(-3, 4, n)).astype(np.float32)
    return np.ascontiguousarray(np.concatenate([p, inten[:, None]], axis=1), np.float32)


@pytest.fixture(scope="module")
def hdl_sweeps(scene):
    from loam_velodyne_b200 import synth
    lidar = synth.Lidar.hdl64()
    out = []
    for i in range(2):
        pts, _ = synth.make_sweep(scene, lidar, i, yaw_rate=math.radians(5.0))
        out.append(registered(pts, 0.3 * i, (-40.0 + 4.1 * i, 0.2 * i, 25.0 - 3.3 * i)))
    return out


def assert_normals(got, keys, cent, counts, radius, vp, drv, what):
    """got = (centroids, counts, normals) of the GPU; keys / cent / counts: the exported cloud it must equal."""
    gc, gn, gnrm = got
    assert gc.shape == cent.shape, f"{what}: {gc.shape} vs {cent.shape}"
    assert np.array_equal(bits(gc), bits(cent)) and np.array_equal(gn, counts), f"{what}: centroids or counts differ"
    ref = nr.normals(keys, cent, radius, vp, drv)
    nan_g, nan_r = np.isnan(gnrm), np.isnan(ref)
    assert np.array_equal(nan_g, nan_r), f"{what}: NaN in {int((nan_g != nan_r).any(axis=1).sum())} other places"
    diff = (bits(gnrm) != bits(ref)).any(axis=1)
    assert not diff.any(), f"{what}: {int(diff.sum())} of {keys.size} normals differ, first {np.nonzero(diff)[0][:5]}"
    return ref


@pytest.mark.parametrize("leaf", [0.05, 0.1, 0.4])
@pytest.mark.parametrize("radius", [1, 2, 3])
def test_inserted_clouds(build_libs, hdl_sweeps, drv, leaf, radius):
    """Box clouds and registered HDL-64E sweeps; viewpoints: the origin, a far point, and exactly on a centroid (the
    flip product of that voxel is exactly 0)."""
    from loam_velodyne_b200 import api
    clouds = [box_cloud(60000, (-3, -1, -3), (3, 1, 3), 1, leaf)] + (hdl_sweeps if leaf > 0.05 else hdl_sweeps[:1])
    ref = dr.DenseMapRef(leaf)
    c = api.Ctx(0)
    try:
        c.dense_enable(leaf)
        for pts in clouds:
            c.cloud_upload(api.C_MAP_FULL, pts)
            c.dense_insert(api.C_MAP_FULL)
            ref.insert(pts)
        cent, counts = c.dense_export()
        rc, rn = ref.export()
        assert np.array_equal(bits(cent), bits(rc)) and np.array_equal(counts, rn)
        on = cent[cent.shape[0] // 3, :3].astype(np.float64)
        for vp in ((0.0, 0.0, 0.0), (1.0e4, -3.0e3, 250.5), tuple(on)):
            got = c.dense_export_normals(None, radius, vp)
            r = assert_normals(got, ref.keys, cent, counts, radius, vp, drv, f"leaf {leaf} radius {radius} vp {vp}")
            assert (~np.isnan(r[:, 0])).sum() > cent.shape[0] // 2
    finally:
        c.close()


@pytest.mark.parametrize("name", list(nr.edge_cases()))
def test_edge_cases(build_libs, drv, name):
    """The key-range edges (the last x index beside the next row, the last y index beside the next plane, the last z
    plane), a lone voxel, two voxels, three collinear voxels with the viewpoint on the middle one, the empty map."""
    from loam_velodyne_b200 import api
    pts, vp, _ = nr.edge_cases()[name]
    ref = dr.DenseMapRef(nr.EDGE_LEAF)
    ref.insert(pts)
    cent, counts = ref.export()
    c = api.Ctx(0)
    try:
        c.dense_enable(nr.EDGE_LEAF)
        c.cloud_upload(api.C_MAP_FULL, pts)
        c.dense_insert(api.C_MAP_FULL)
        for radius in (1, 2, 3):
            for ratio in (None, 1.0):
                assert_normals(c.dense_export_normals(ratio, radius, vp), ref.keys, cent, counts, radius, vp, drv,
                               f"{name} radius {radius}")
    finally:
        c.close()


def test_filtered_voxels(build_libs, scene, drv):
    """Evidence from dense_observe: at ratios 0, 1 and +inf the export with normals keeps exactly the voxels of
    dense_export(ratio), and a filtered voxel neither gets a normal nor changes its neighbours' normals."""
    from loam_velodyne_b200 import api, synth
    import visibility_reference as vr
    run = vr.moving_box_run(scene, synth.Lidar.vlp16(), 10)
    leaf = 0.1
    ref = dr.DenseMapRef(leaf)
    c = api.Ctx(0)
    try:
        c.dense_enable(leaf)
        c.dense_visibility(1.0, 2.0, 0.5)
        for pts, twist, _ in run:
            c.cloud_upload(api.C_MAP_FULL, pts)
            c.dense_observe(api.C_MAP_FULL, twist)
            c.dense_insert(api.C_MAP_FULL)
            ref.insert(pts)
        cent, counts, hits, misses = c.dense_export(math.inf, evidence=True)
        assert np.array_equal(bits(cent), bits(ref.export()[0]))
        vp = (0.5, 1.0, -2.0)
        for ratio in (0.0, 1.0, math.inf):
            keep = misses.astype(np.float64) <= ratio * hits.astype(np.float64)
            fc, fn = c.dense_export(ratio)
            assert np.array_equal(bits(fc), bits(cent[keep])) and np.array_equal(fn, counts[keep])
            right = assert_normals(c.dense_export_normals(ratio, 2, vp), ref.keys[keep], cent[keep], counts[keep], 2,
                                   vp, drv, f"ratio {ratio}")
            if ratio < math.inf:
                assert (~keep).sum() > 100
                wrong = nr.normals(ref.keys, cent, 2, vp, drv)[keep]
                assert (bits(right) != bits(wrong)).any(axis=1).sum() > 10
    finally:
        c.close()


def test_errors_and_capacity(build_libs):
    import ctypes as C
    from loam_velodyne_b200 import api
    c = api.Ctx(0)
    try:
        assert c.dense_export_normals()[0].shape == (0, 4)  # map off: nothing exported
        c.dense_enable(0.2)
        pts = box_cloud(5000, (-1, -1, -1), (1, 1, 1), 3, 0.2)
        c.cloud_upload(api.C_MAP_FULL, pts)
        c.dense_insert(api.C_MAP_FULL)
        for ratio, radius, vp in ((None, 0, (0, 0, 0)), (None, 4, (0, 0, 0)), (float("nan"), 1, (0, 0, 0)),
                                  (-1.0, 1, (0, 0, 0)), (None, 1, (float("nan"), 0, 0)), (None, 1, (0, float("inf"), 0)),
                                  (None, 1, (0, 0, -float("inf")))):
            with pytest.raises(api.LoamB200Error, match="invalid argument"):
                c.dense_export_normals(ratio, radius, vp)
        n = c.dense_stats()["voxels"]
        xyzi = np.zeros((n, 4), np.float32)
        nrm = np.zeros((n, 4), np.float32)
        got = C.c_int(0)
        vp = (C.c_double * 3)(0.0, 0.0, 0.0)
        L = c.L
        assert L.loam_b200_dense_export_normals(c.h, math.inf, 1, None, api._fp(xyzi), None, api._fp(nrm), n,
                                                C.byref(got)) == ERR_ARG
        assert L.loam_b200_dense_export_normals(c.h, math.inf, 1, vp, api._fp(xyzi), None, api._fp(nrm), n - 1,
                                                C.byref(got)) == ERR_CAPACITY and got.value == n
        assert L.loam_b200_dense_export_normals(c.h, math.inf, 1, vp, api._fp(xyzi), None, None, n,
                                                C.byref(got)) == ERR_ARG
        assert L.loam_b200_dense_export_normals(c.h, math.inf, 1, vp, api._fp(xyzi), None, api._fp(nrm), n,
                                                C.byref(got)) == 0 and got.value == n
        ref = c.dense_export_normals(None, 1, (0, 0, 0))
        assert np.array_equal(bits(xyzi), bits(ref[0])) and np.array_equal(bits(nrm), bits(ref[2]))
        c.dense_clear()
        assert c.dense_export_normals(1.0, 3, (1, 2, 3))[0].shape == (0, 4)
    finally:
        c.close()


SUMS = [(0.01, 1.3, -0.02, 0.3, 0.1, 0.2), (-0.02, 2.4, 0.03, 24.9, 0.5, 24.8), (0.0, -1.1, 0.0, -74.9, 0.2, -25.1),
        (0.03, 3.0, -0.01, -380.0, 1.0, 10.0), (0.0, -2.9, 0.02, 380.0, -1.0, -30.0), (0.0, 0.4, 0.0, -5.0, 0.0, 3.0)]
SUMS += [(0.0, 0.05 * i, 0.0, 0.4 * i, 0.02 * i, 0.9 * i) for i in range(16)]


def test_mapping_stage(build_libs, scene, map_200k, drv):
    """VLP-16 through the mapping stage with the dense map and the visibility pass on: LaserMapping.dense_map_normals
    equals the restatement applied to dense_map(max_miss_ratio=1, evidence=True)."""
    from loam_velodyne_b200 import api, synth
    reg = api.ScanRegistration()
    m = api.LaserMapping(0.1, 10)
    m.seed(*map_200k)
    m.enable_dense_map(0.1)
    m.enable_dense_visibility(1.0, 2.0, 1.0)
    lidar = synth.Lidar.vlp16(n_az=900)
    ref = dr.DenseMapRef(0.1)
    for it, sum6 in enumerate(SUMS):
        pts, rs = synth.make_sweep(scene, lidar, it, yaw_rate=math.radians(5.0))
        reg.process(pts, rs)
        m.set_inputs(reg.cloud("less_sharp"), reg.cloud("less_flat"), pts)
        m.update_odometry(np.asarray(sum6, np.float32))
        assert m.process()
        ref.insert(m.cloud("full"))
    cent, counts, hits, misses = m.dense_map(math.inf, evidence=True)
    assert np.array_equal(bits(cent), bits(ref.export()[0])) and cent.shape[0] > 10000
    keep = misses.astype(np.float64) <= hits.astype(np.float64)
    kc, kn, _, _ = m.dense_map(1.0, evidence=True)
    assert np.array_equal(bits(kc), bits(cent[keep])) and np.array_equal(kn, counts[keep]) and (~keep).any()
    for radius, vp in ((1, (0.0, 0.0, 0.0)), (2, (3.5, 1.0, -12.25))):
        assert_normals(m.dense_map_normals(1.0, radius, vp), ref.keys[keep], kc, kn, radius, vp, drv,
                       f"mapping stage radius {radius}")
