"""Distance field of the whole-run voxel map on the GPU (csrc/densemap.cuh: dense_edt_*_kernel,
dense_distance_query_kernel; loam_b200_dense_distance_build / _query) against the numpy restatement
(tests/distance_reference.py): sq exactly, dist and the query's distance and gradient by float bits, on hand-made
targets, targets built on the GPU at three leaves from two sensors, host and device queries; the lifecycle, the error
paths and limits, launch counts, and the drop-in path on the mapping stage's own map."""
import math

import numpy as np
import pytest

import align_reference as ar
import dense_reference as dr
import distance_reference as dist_ref
from test_align_reference import HELD_OUT, MAP_TWISTS, lidars
from test_dense_align import map_ctx
from test_distance_reference import LIMIT_CASES

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same(a, b):
    """Float bits equal, NaN equal to NaN."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(bits(a[~na]), bits(b[~nb]))


def load_voxels(c, leaf, vox):
    """Load a target of the voxels (their centres; every other one without a normal) -> its keys."""
    cent = dist_ref.centres(leaf, vox)
    nrm = np.tile(np.float32([0, 1, 0, 0]), (cent.shape[0], 1))
    nrm[1::2] = np.nan
    keys = dr.voxel_keys(cent, leaf)
    assert np.array_equal(np.sort(keys), np.sort(dist_ref.keys_of_voxels(vox)))
    c.dense_target_load(leaf, cent, nrm)
    return keys


def assert_field(fn, keys, leaf, lo, dims, md, what):
    dist, sq = fn(lo, dims, md)
    wd, ws = dist_ref.field(keys, leaf, lo, dims, md)
    assert sq.shape == ws.shape, what
    assert np.array_equal(sq, ws), f"{what}: {int((sq != ws).sum())} of {sq.size} sq differ"
    assert same(dist, wd), f"{what}: dist differs"
    return sq


def query_points(leaf, lo, dims, seed, n=4000):
    """Points over the box's cells and one cell beyond it, its first and last centres and their neighbours 1 ulp and
    half a cell outside, and non-finite points."""
    rng = np.random.RandomState(seed)
    L = float(np.float32(leaf))
    lo = np.asarray(lo, np.float64)
    dims = np.asarray(dims, np.float64)
    p = (lo + rng.uniform(-1.0, dims + 1.0, (n, 3))) * L
    first = (lo + 0.5) * L
    last = (lo + dims - 0.5) * L
    extra = [first, last]
    for c, s in ((first, -1.0), (last, 1.0)):
        for ax in range(3):
            for off in (0.0, 0.5 * L):
                q = np.array(c, np.float32)
                q[ax] = np.nextafter(np.float32(c[ax] + s * off), np.float32(s * np.inf))
                extra.append(q)
    pts = np.concatenate([p, np.array(extra, np.float64)]).astype(np.float32)
    pts = np.concatenate([pts, np.ones((pts.shape[0], 1), np.float32)], axis=1)
    pts[::97, 1] = np.nan
    pts[5::211, 0] = np.inf
    pts[7::211, 2] = -np.inf
    return np.ascontiguousarray(pts)


def assert_query(fn, sq, leaf, lo, md, pts, what):
    d, g = fn(pts)
    wd, wg = dist_ref.query(sq, leaf, lo, md, pts)
    assert same(d, wd), f"{what}: {int((bits(d) != bits(wd)).sum())} of {d.size} distances differ"
    assert same(g, wg), f"{what}: gradients differ"
    return d, g


@pytest.mark.parametrize("name", list(dist_ref.edge_cases()))
def test_edge_cases(build_libs, name):
    """The hand-made targets, loaded into a context without the map: brick faces and corners, negative indices, an
    obstacle only in the pad, a cell at exactly max_distance, boxes one cell thick."""
    from loam_velodyne_b200 import api
    leaf, vox, lo, dims, md = dist_ref.edge_cases()[name]
    c = api.Ctx(0)
    try:
        keys = load_voxels(c, leaf, vox)
        sq = assert_field(c.dense_distance_field, keys, leaf, lo, dims, md, name)
        pts = query_points(leaf, lo, dims, seed=len(name))
        d, _ = assert_query(lambda p: c.dense_distance_query(p, gradient=True), sq, leaf, lo, md, pts, name)
        if min(dims) >= 2:
            assert np.isfinite(d).sum() > 100
        else:
            assert np.isnan(d).all()
    finally:
        c.close()


def test_empty_target(build_libs):
    """An empty target: beyond everywhere, no ray index, nothing launched; queries saturate."""
    from loam_velodyne_b200 import api
    c = api.Ctx(0)
    try:
        c.dense_target_load(0.25, np.zeros((0, 4), np.float32), np.zeros((0, 4), np.float32))
        before = c.launch_count()
        dist, sq = c.dense_distance_field((-3, -2, -1), (7, 5, 4), 1.0)
        assert (sq == -1).all() and np.isinf(dist).all() and sq.shape == (4, 5, 7)
        assert c.launch_count() == before and c.dense_ray_index_bytes() == 0
        d = c.dense_distance_query(dist_ref.centres(0.25, [[0, 0, 0], [-3, -2, -1], [3, 2, 2]]))
        assert (d == np.float32(1.0)).all()
    finally:
        c.close()


BOXES = [((-4.0, -2.0, -4.0), (4.0, 1.5, 4.0)), ((1.3, -2.4, -7.2), (9.6, 1.1, -0.3))]  # both hold ground


@pytest.mark.parametrize("leaf", [0.1, 0.2, 0.4])
@pytest.mark.parametrize("sensor", ["vlp16", "hdl64"])
def test_built_targets(build_libs, scene, sensor, leaf):
    """Targets built on the GPU from the map sweeps; boxes around them at several max_distance; host queries."""
    from loam_velodyne_b200 import api
    lidar = lidars()[sensor]
    c, ref = map_ctx(scene, lidar, leaf)
    try:
        n = c.dense_target_build(None, 2, (0.5, 1.0, -2.0))
        keys = ref.keys
        assert n == keys.size
        for b, (mn, mx) in enumerate(BOXES):
            shift = np.asarray(MAP_TWISTS[b % len(MAP_TWISTS)][3:], np.float64)
            lo, dims = api.voxel_box(np.add(mn, shift), np.add(mx, shift), leaf)
            for md in (0.5, 1.3, 3.0):
                what = f"{sensor} leaf {leaf} box {b} max {md}"
                sq = assert_field(c.dense_distance_field, keys, leaf, lo, dims, md, what)
                assert (sq == 0).any() and (sq > 0).any()
                pts = query_points(leaf, lo, dims, seed=b)
                assert_query(lambda p: c.dense_distance_query(p, gradient=True), sq, leaf, lo, md, pts, what)
    finally:
        c.close()


def test_sources_lifecycle_and_launches(build_libs, scene):
    """Host and device queries give the same bits, with or without the gradient; the field is a snapshot (later
    inserts change nothing), the next build replaces it, a target rebuild or load drops it; launches count under the
    dense family: the first field after a target build also builds the ray index."""
    import torch
    from loam_velodyne_b200 import api, synth
    lidar = lidars()["hdl64"]
    leaf = 0.2
    c, ref = map_ctx(scene, lidar, leaf)
    try:
        c.dense_target_build(None, 2, (0.0, 0.0, 0.0))
        assert c.dense_distance_bytes() == 0
        lo, dims = api.voxel_box((-5.0, -2.0, -5.0), (5.0, 2.0, 5.0), leaf)
        c.profile(True)
        dist, sq = c.dense_distance_field(lo, dims, 2.0)
        prof = c.profile_get()
        assert prof["dense"][1] >= 3 + 4 and sum(v[1] for k, v in prof.items() if k != "dense") == 0
        assert c.dense_distance_bytes() == 4 * sq.size and c.dense_ray_index_bytes() > 0
        c.profile(True)
        before = c.launch_count()
        again = c.dense_distance_field(lo, dims, 2.0, download=False)
        assert again == (None, None)
        assert c.launch_count() - before == 3 and c.profile_get()["dense"][1] == 3
        pts = query_points(leaf, lo, dims, seed=3, n=20000)
        before = c.launch_count()
        d, g = c.dense_distance_query(pts, gradient=True)
        assert c.launch_count() - before == 1
        assert same(c.dense_distance_query(pts), d)
        dev = torch.from_numpy(pts).cuda()
        dd, dg = c.dense_distance_query(dev.data_ptr(), on_device=True, n=pts.shape[0], gradient=True)
        torch.cuda.synchronize()
        assert same(dd, d) and same(dg, g)
        wd, wg = dist_ref.query(sq, leaf, lo, 2.0, pts)
        assert same(d, wd) and same(g, wg)
        # snapshot: an insert after the build changes nothing
        extra = ar.static_sweep(scene, synth.Lidar.hdl64(512), HELD_OUT[2].astype(np.float64) + 0.5, seed=7)[1]
        c.cloud_upload(api.C_MAP_FULL, extra)
        c.dense_insert(api.C_MAP_FULL)
        assert same(c.dense_distance_query(pts), d)
        # the next build replaces it
        lo2, dims2 = api.voxel_box((-2.0, -1.0, -2.0), (3.0, 1.0, 2.0), leaf)
        _, sq2 = c.dense_distance_field(lo2, dims2, 0.6)
        assert_query(lambda p: c.dense_distance_query(p, gradient=True), sq2, leaf, lo2, 0.6, pts, "replaced")
        assert c.dense_distance_bytes() == 4 * sq2.size
        # a target rebuild drops it; the new field sees the extra sweep
        c.dense_target_build(None, 2, (0.0, 0.0, 0.0))
        assert c.dense_distance_bytes() == 0
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_distance_query(pts)
        ref.insert(extra)
        assert_field(c.dense_distance_field, ref.keys, leaf, lo, dims, 2.0, "after the rebuild")
        # a load drops it
        load_voxels(c, leaf, [[0, 0, 0]])
        assert c.dense_distance_bytes() == 0
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_distance_query(pts)
    finally:
        c.close()


def test_errors_and_limits(build_libs, scene):
    import ctypes as C
    from loam_velodyne_b200 import api, synth
    c = api.Ctx(0)
    try:
        pts = dist_ref.centres(0.5, [[0, 0, 0]])
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_distance_field((0, 0, 0), (2, 2, 2), 1.0)  # no target
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_distance_query(pts)
        for leaf in sorted({case[0] for case in LIMIT_CASES}):
            load_voxels(c, leaf, [[1, 2, 3]])
            with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
                c.dense_distance_query(pts)  # a target without a field
            for cl, lo, dims, md, ok in LIMIT_CASES:
                if cl != leaf:
                    continue
                assert dist_ref.box_ok(leaf, lo, dims, md) == ok
                if ok:
                    c.dense_distance_field(lo, dims, md, download=False)
                else:
                    with pytest.raises(api.LoamB200Error, match="invalid argument"):
                        c.dense_distance_field(lo, dims, md, download=False)
        load_voxels(c, 0.5, [[1, 2, 3]])
        for lo, dims, md in (((0, 0, 0), (2, 2, 2), float("nan")), ((0, 0, 0), (2, 2, 2), -1.0),
                             ((0, 0, 0), (2, -1, 2), 1.0), ((0, 0, 0), (8192, 1, 1), 0.25)):
            with pytest.raises(api.LoamB200Error, match="invalid argument"):
                c.dense_distance_field(lo, dims, md)
        # a failed build leaves no field
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_distance_query(pts)
        L = c.L
        lo = np.zeros(3, np.int32)
        dims = np.full(3, 2, np.int32)
        assert L.loam_b200_dense_distance_build(c.h, None, api._ip(dims), 1.0, None, None) == -1
        assert L.loam_b200_dense_distance_build(c.h, api._ip(lo), None, 1.0, None, None) == -1
        assert L.loam_b200_dense_distance_build(c.h, api._ip(lo), api._ip(dims), 1.0, None, None) == 0
        out = np.zeros(4, np.float32)
        assert L.loam_b200_dense_distance_query(c.h, None, 1, 0, api._fp(out), None) == -1
        assert L.loam_b200_dense_distance_query(c.h, api._fp(pts), 1, 0, None, None) == -1
        assert L.loam_b200_dense_distance_query(c.h, api._fp(pts), -1, 0, api._fp(out), None) == -1
        before = c.launch_count()
        assert L.loam_b200_dense_distance_query(c.h, None, 0, 0, None, None) == 0
        assert c.launch_count() == before
    finally:
        c.close()
    lidar = synth.Lidar.vlp16()
    sweeps = [synth.make_sweep(scene, lidar, i, yaw_rate=math.radians(5.0)) for i in range(3)]
    pl = api.Pipeline()
    pl.mapping.enable_dense_map(0.1)
    for q, rs in sweeps:
        pl.submit(q, rs)
    with pytest.raises(api.LoamB200Error, match="in flight"):
        pl.mapping.build_dense_distance_field((0, 0, 0), (4, 4, 4), 1.0)
    with pytest.raises(api.LoamB200Error, match="in flight"):
        pl.mapping.query_dense_distance(dist_ref.centres(0.1, [[0, 0, 0]]))
    while pl.collect(wait=True) is not None:
        pass
    assert pl.mapping.build_dense_target() > 0
    cent = pl.mapping.dense_map_normals(None, 2, (0.0, 0.0, 0.0))[0]
    keys = dr.voxel_keys(cent, 0.1)
    lo = dist_ref.target_voxels(keys[:1])[0] - 10
    sq = assert_field(pl.mapping.build_dense_distance_field, keys, 0.1, lo, (20, 20, 20), 1.0, "pipeline")
    assert (sq == 0).any()
    pl.sync()


def test_unused_launches_nothing(build_libs, scene):
    """With the feature unused nothing is launched for it: a target build and a ray cast launch what they did."""
    from loam_velodyne_b200 import api
    c, _ = map_ctx(scene, lidars()["vlp16"], 0.2)
    try:
        c.dense_target_build(None, 2, (0.0, 0.0, 0.0))
        assert c.dense_distance_bytes() == 0
        c.dense_raycast(api.lidar_rays([0.0], 64), np.zeros(6, np.float32), 0.0, 50.0)
        before = c.launch_count()
        c.dense_raycast(api.lidar_rays([0.0], 64), np.zeros(6, np.float32), 0.0, 50.0)
        assert c.launch_count() - before == 1 and c.dense_distance_bytes() == 0
    finally:
        c.close()


SUMS = [(0.0, 0.05 * i, 0.0, 0.4 * i, 0.02 * i, 0.9 * i) for i in range(8)]


def test_mapping_stage(build_libs, scene, map_200k):
    """VLP-16 through the mapping stage with the dense map on: the drop-in field and queries equal the Ctx path on a
    target loaded from the export, and both equal the restatement."""
    from loam_velodyne_b200 import api, synth
    reg = api.ScanRegistration()
    m = api.LaserMapping(0.1, 10)
    m.seed(*map_200k)
    m.enable_dense_map(0.1)
    lidar = synth.Lidar.vlp16(n_az=900)
    for it, sum6 in enumerate(SUMS):
        pts, rs = synth.make_sweep(scene, lidar, it, yaw_rate=math.radians(5.0))
        reg.process(pts, rs)
        m.set_inputs(reg.cloud("less_sharp"), reg.cloud("less_flat"), pts)
        m.update_odometry(np.asarray(sum6, np.float32))
        assert m.process()
    vp = (0.0, 0.0, 0.0)
    n = m.build_dense_target(None, 2, vp)
    cent, _, nrm = m.dense_map_normals(None, 2, vp)
    assert n == cent.shape[0] > 10000
    keys = dr.voxel_keys(cent, 0.1)
    lo, dims = api.voxel_box((-6.0, -2.5, -6.0), (6.0, 1.5, 6.0), 0.1)
    c = api.Ctx(0)
    try:
        c.dense_target_load(0.1, cent, nrm)
        assert_field(m.build_dense_distance_field, keys, 0.1, lo, dims, 1.5, "drop-in")
        cd, csq = c.dense_distance_field(lo, dims, 1.5)
        md, msq = m.build_dense_distance_field(lo, dims, 1.5)
        assert np.array_equal(csq, msq) and same(cd, md)
        pts = query_points(0.1, lo, dims, seed=9, n=50000)
        got = assert_query(lambda p: m.query_dense_distance(p, gradient=True), msq, 0.1, lo, 1.5, pts, "drop-in")
        want = c.dense_distance_query(pts, gradient=True)
        assert same(got[0], want[0]) and same(got[1], want[1])
        assert same(m.query_dense_distance(pts), got[0])
        frac = np.isfinite(got[0]).mean()
        print(f"defined share {frac:.3f}, within range {(got[0][np.isfinite(got[0])] < 1.5).mean():.3f}")
    finally:
        c.close()
