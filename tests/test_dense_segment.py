"""Euclidean segmentation on the GPU (csrc/densemap.cuh: dense_seg_*_kernel; loam_b200_dense_segment /
loam_b200_cloud_segment) against the numpy restatement (tests/segment_reference.py): labels and segment records bit
for bit on hand-made clouds and targets, targets built on the GPU at three leaves and three tolerances, a saved and
reloaded target, sweeps from host and device memory with NaNs, and the union-find's worst cases run twice; then the
errors, the capacity rule, launch counts, the untouched target products and the drop-in path."""
import numpy as np
import pytest

import align_reference as ar
import segment_reference as sr
from test_align_reference import HELD_OUT, lidars
from test_dense_align import map_ctx
from test_segment_reference import cloud, edge_case_clouds, target_cases

pytestmark = pytest.mark.gpu


def assert_same(got, want, what):
    gl, gs = got
    wl, ws = want
    assert np.array_equal(gl, wl), f"{what}: {int((gl != wl).sum())} of {gl.size} labels differ"
    assert set(gs) == set(ws)
    for f in ws:
        assert gs[f].shape == ws[f].shape, f"{what}: {f} shape {gs[f].shape} vs {ws[f].shape}"
        assert np.array_equal(gs[f].view(np.uint8), ws[f].view(np.uint8)), f"{what}: {f} differs"


def load_target(c, leaf, pts):
    keys, cent = sr.target_of(pts, leaf)
    c.dense_target_load(leaf, cent, np.tile(np.float32([0, 1, 0, 0]), (cent.shape[0], 1)))
    return keys, cent


@pytest.mark.parametrize("name", list(edge_case_clouds()))
def test_hand_made_clouds(build_libs, name):
    from loam_velodyne_b200 import api
    pts, tol, mn, mx = edge_case_clouds()[name]
    c = api.Ctx(0)
    try:
        assert_same(c.segment_cloud(pts, tol, mn, None if mx == sr.INT_MAX else mx), sr.cloud_segment(pts, tol, mn, mx),
                    name)
    finally:
        c.close()


def test_hand_made_targets(build_libs):
    """Hand-made targets loaded from the host, and the same points as a cloud at cell = tol in key order."""
    from loam_velodyne_b200 import api
    c = api.Ctx(0)
    try:
        for name, (leaf, pts, tol) in target_cases().items():
            keys, cent = load_target(c, leaf, pts)
            assert_same(c.dense_segment(tol), sr.target_segment(keys, cent, leaf, tol), name)
        rng = np.random.RandomState(11)
        v = np.unique(rng.randint(-30, 30, (3000, 3)), axis=0)
        pts = cloud((v + rng.uniform(0.05, 0.95, v.shape)) * 0.25)
        keys, cent = load_target(c, 0.25, pts)
        want = sr.target_segment(keys, cent, 0.25, 0.25)
        assert_same(c.dense_segment(0.25), want, "one point per voxel")
        assert_same(c.segment_cloud(cent, 0.25), want, "as a cloud")
    finally:
        c.close()


@pytest.mark.parametrize("leaf", [0.1, 0.2, 0.4])
def test_built_targets(build_libs, scene, leaf):
    """Targets built on the GPU from HDL-64E map sweeps at tol = 1.5, 2.5 and 4 leaves, with size filters; then the
    target saved through the export and loaded back."""
    from loam_velodyne_b200 import synth
    c, ref = map_ctx(scene, synth.Lidar.hdl64(512), leaf)
    try:
        n = c.dense_target_build(None, 2, (0.0, 0.0, 0.0))
        cent = ref.export()[0]
        assert n == ref.keys.size
        for mult, mn, mx in ((1.5, 1, None), (2.5, 3, 5000), (4.0, 1, None)):
            tol = float(np.float32(mult * leaf))
            want = sr.target_segment(ref.keys, cent, leaf, tol, mn, sr.INT_MAX if mx is None else mx)
            got = c.dense_segment(tol, mn, mx)
            assert_same(got, want, f"leaf {leaf} tol {tol}")
            assert got[1]["size"].size > 1 and (got[0] >= 0).any()
        saved_c, _, saved_n = c.dense_export_normals(None, 2, (0.0, 0.0, 0.0))
        c.dense_target_load(leaf, saved_c, saved_n)
        keys, loaded = sr.target_of(saved_c, leaf)
        tol = float(np.float32(2.5 * leaf))
        assert_same(c.dense_segment(tol), sr.target_segment(keys, loaded, leaf, tol), "reloaded")
    finally:
        c.close()


def test_sweeps_from_host_and_device(build_libs, scene):
    import torch
    from loam_velodyne_b200 import api, synth
    c = api.Ctx(0)
    try:
        for k, (lidar, tol) in enumerate(((synth.Lidar.vlp16(), 0.5), (synth.Lidar.hdl64(1024), 0.3))):
            pts = ar.static_sweep(scene, lidar, HELD_OUT[k].astype(np.float64), seed=40 + k)[0]
            pts[::97, 1] = np.nan
            pts[5::211, 0] = np.inf
            want = sr.cloud_segment(pts, tol, 2)
            got = c.segment_cloud(pts, tol, 2)
            assert_same(got, want, f"host {k}")
            assert got[1]["size"].size > 5
            dev = torch.from_numpy(pts).cuda()
            assert_same(c.segment_cloud(dev.data_ptr(), tol, 2, on_device=True, n=pts.shape[0]), want, f"device {k}")
    finally:
        c.close()


def ground_plane(leaf):
    """A 400 x 300 voxel floor (120 000 voxels, one component at tol = 1.5 leaves: every hook lands on one root)."""
    g = np.stack(np.meshgrid(np.arange(400), np.arange(300), indexing="ij"), -1).reshape(-1, 2)
    return cloud(np.stack([(g[:, 0] + 0.5) * leaf, np.full(g.shape[0], 0.5 * leaf), (g[:, 1] + 0.5) * leaf], 1))


def spiral(tol, n=60000):
    """A long thin spiral, points 0.6 tol apart: one component that is a single long chain."""
    s = np.arange(n, dtype=np.float64) * 0.6 * tol
    r = 2.0 + s / 200.0
    th = s / r
    return cloud(np.stack([r * np.cos(th), 0.01 * s, r * np.sin(th)], 1))


def test_union_find_worst_cases(build_libs):
    """Contention on one root (a ground plane) and deep chains (a spiral), each twice: same bits both times."""
    from loam_velodyne_b200 import api
    c = api.Ctx(0)
    try:
        leaf = 0.1
        keys, cent = load_target(c, leaf, ground_plane(leaf))
        want = sr.target_segment(keys, cent, leaf, 0.15)
        assert want[1]["size"].tolist() == [120000]
        for _ in range(2):
            assert_same(c.dense_segment(0.15), want, "ground plane")
        pts = spiral(0.2)
        want = sr.cloud_segment(pts, 0.2)
        assert want[1]["size"].tolist() == [pts.shape[0]]
        perm = np.random.RandomState(3).permutation(pts.shape[0])
        want_p = sr.cloud_segment(pts[perm], 0.2)
        for _ in range(2):
            assert_same(c.segment_cloud(pts, 0.2), want, "spiral")
            assert_same(c.segment_cloud(pts[perm], 0.2), want_p, "shuffled spiral")
    finally:
        c.close()


def test_errors_capacity_launches_and_products(build_libs, scene):
    """Refused calls change nothing; the capacity rule; a fixed launch count per entry count under the dense family;
    ray cast, distance field and alignment give the same bits before and after a segmentation."""
    import ctypes as C
    from loam_velodyne_b200 import api, synth
    leaf = 0.2
    c = api.Ctx(0)
    try:
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_segment(0.3)  # no target
        pts = edge_case_clouds()["filters"][0]
        for args in ((float("nan"),), (0.0,), (-1.0,), (float("inf"),), (0.5, 0), (0.5, 3, 2)):
            with pytest.raises(api.LoamB200Error, match="invalid argument"):
                c.segment_cloud(pts, *args)
    finally:
        c.close()
    c, ref = map_ctx(scene, synth.Lidar.vlp16(), leaf)
    try:
        n = c.dense_target_build(None, 2, (0.0, 0.0, 0.0))
        sweep = ar.static_sweep(scene, synth.Lidar.vlp16(), HELD_OUT[0].astype(np.float64), seed=70)[0]
        lo, dims = api.voxel_box((-4.0, -2.0, -4.0), (4.0, 1.5, 4.0), leaf)
        rays = api.lidar_rays([-10.0, 0.0, 10.0], 256)

        def products():
            r = c.dense_raycast(rays, HELD_OUT[0], 0.0, 50.0)
            d = c.dense_distance_field(lo, dims, 1.0)
            a = c.dense_align(sweep, HELD_OUT[0], 1, 5)
            return [r[0], r[1], d[0], d[1], a[0]]

        before = products()
        want = sr.target_segment(ref.keys, ref.export()[0], leaf, 0.5)
        c.profile(True)
        l0 = c.launch_count()
        got = c.dense_segment(0.5)
        launches = c.launch_count() - l0
        prof = c.profile_get()
        assert prof["dense"][1] == launches and sum(v[1] for k, v in prof.items() if k != "dense") == 0
        assert_same(got, want, "first")
        for tol in (float(np.float32(4 * leaf)) * 1.001, 1.0, float("nan")):
            with pytest.raises(api.LoamB200Error, match="invalid argument"):
                c.dense_segment(tol)
        K = got[1]["size"].size
        seg = (api.Segment * 4)()
        k = C.c_int(0)
        assert c.L.loam_b200_dense_segment(c.h, 0.5, 1, 2**31 - 1, None, seg, 3, C.byref(k)) == -5  # ERR_CAPACITY
        assert k.value == K > 3
        assert c.L.loam_b200_dense_segment(c.h, 0.5, 1, 2**31 - 1, None, None, 0, C.byref(k)) == -5 and k.value == K
        assert c.L.loam_b200_dense_segment(c.h, 0.5, 1, 2**31 - 1, None, None, 1, C.byref(k)) == -1
        assert c.L.loam_b200_dense_segment(c.h, 0.5, 1, 2**31 - 1, None, seg, 4, None) == -1
        assert c.L.loam_b200_dense_segment(c.h, 0.5, 1, 2**31 - 1, None, seg, -1, C.byref(k)) == -1
        assert_same(c.dense_segment(0.5), want, "after the refusals")
        # the launch count depends on the entry count only: a different target of the same size launches the same
        c2 = api.Ctx(0)
        try:
            assert n <= 120000
            load_target(c2, leaf, ground_plane(leaf)[:n])
            l0 = c2.launch_count()
            c2.dense_segment(0.5, 2, 100)
            assert c2.launch_count() - l0 == launches
            l0 = c2.launch_count()
            c2.segment_cloud(sweep, 0.5)
            cloud_launches = c2.launch_count() - l0
            l0 = c2.launch_count()
            c2.segment_cloud(np.ascontiguousarray(sweep[::-1]), 0.5, 3)
            assert c2.launch_count() - l0 == cloud_launches
            l0 = c2.launch_count()
            c2.segment_cloud(np.zeros((0, 4), np.float32), 0.5)
            c2.dense_target_load(leaf, np.zeros((0, 4), np.float32), np.zeros((0, 4), np.float32))
            assert c2.dense_segment(0.5)[1]["size"].size == 0
            assert c2.launch_count() == l0
        finally:
            c2.close()
        after = products()
        for a, b in zip(before, after):
            assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
    finally:
        c.close()


def test_drop_in_equals_ctx(build_libs, scene):
    """LaserMapping.segment_dense_target (BasicLaserMapping::segmentDenseTarget) equals Ctx.dense_segment."""
    from loam_velodyne_b200 import api, synth
    c, ref = map_ctx(scene, lidars()["vlp16"], 0.1)
    try:
        c.dense_target_build(None, 2, (0.0, 0.0, 0.0))
        cent, _, nrm = c.dense_export_normals(None, 2, (0.0, 0.0, 0.0))
        m = api.LaserMapping(0.1, 10)
        m.load_dense_target(0.1, cent, nrm)
        for tol, mn, mx in ((0.15, 1, None), (0.3, 5, 2000)):
            assert_same(m.segment_dense_target(tol, mn, mx), c.dense_segment(tol, mn, mx), f"tol {tol}")
        with pytest.raises(api.LoamB200Error):
            m.segment_dense_target(0.5)  # tol / leaf > 4
    finally:
        c.close()


def test_segment_after_refused_target_calls(build_libs):
    """A refused target build or load keeps the target it found (or none, for a load refused on the device): the
    labels are sized from the library's target, never from a copy of an earlier call's count."""
    from loam_velodyne_b200 import api
    leaf = 0.2
    pts = ground_plane(leaf)[::7]
    pts[::3, 1] = np.float32(1.5)  # a few separate pieces
    keys, cent = sr.target_of(pts, leaf)
    nrm = np.tile(np.float32([0, 1, 0, 0]), (cent.shape[0], 1))
    wants = {mn: sr.target_segment(keys, cent, leaf, 0.3, mn) for mn in (1, 10**6)}
    assert wants[10**6][1]["size"].size == 0 and wants[1][1]["size"].size > 1
    c = api.Ctx(0)
    try:
        c.dense_target_load(leaf, cent, nrm)
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_target_build(None, 2)  # no map: refused before the target is touched
        with pytest.raises(api.LoamB200Error, match="invalid argument"):
            c.dense_target_load(float("nan"), cent, nrm)  # refused on the host: the target stays
        assert c.dense_target_size() == cent.shape[0]
        for mn, want in wants.items():
            got = c.dense_segment(0.3, mn)
            assert got[0].size == cent.shape[0]
            assert_same(got, want, f"Ctx min_size {mn}")
        with pytest.raises(api.LoamB200Error, match="invalid argument"):
            c.dense_target_load(leaf, np.concatenate([cent[:1], cent[:1]]), nrm[:2])  # two in one voxel: no target
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_target_size()
        with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
            c.dense_segment(0.3)
    finally:
        c.close()
    m = api.LaserMapping(0.1, 10)
    m.load_dense_target(leaf, cent, nrm)
    with pytest.raises(api.LoamB200Error):
        m.build_dense_target()  # no whole-run map on this object
    with pytest.raises(api.LoamB200Error):
        m.load_dense_target(float("nan"), cent, nrm)
    for mn, want in wants.items():
        assert_same(m.segment_dense_target(0.3, mn), want, f"drop-in min_size {mn}")
