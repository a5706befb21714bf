"""The ground of the whole-run voxel map on the GPU (csrc/densemap.cuh: dense_ground_*_kernel; loam_b200_dense_ground
/ _segment_above_ground / _ground_cloud) against the numpy restatement (tests/ground_reference.py), bit for bit: the
hand-made targets and clouds, targets built at three leaves and one reloaded, the 120 000-voxel floor twice,
segmentation above the ground at three tolerances and its identity with dense_segment, sweeps from host and device
memory into cloud_segment; then errors, the capacity rule, launch counts, the untouched products and the drop-in
path."""
import ctypes as C

import numpy as np
import pytest

import align_reference as ar
import ground_reference as gr
import segment_reference as sr
from test_align_reference import HELD_OUT
from test_dense_align import map_ctx
from test_dense_segment import assert_same, ground_plane
from test_ground_reference import IDENTITY, cloud_case, poles_on_floor, target_cases

pytestmark = pytest.mark.gpu


def load(c, t):
    c.dense_target_load(float(t.leaf), t.cent, t.nrm)


def assert_ground(c, t, prm, what):
    lab, seg, g = gr.dense_ground(t.keys, t.cent, t.nrm, float(t.leaf), prm)
    assert_same(c.dense_ground(prm.ctypes()), (lab, seg), what)
    return g


def test_hand_made(build_libs):
    from loam_velodyne_b200 import api
    c = api.Ctx(0)
    try:
        for name, (t, prm, _) in target_cases().items():
            load(c, t)
            assert_ground(c, t, prm, name)
        t = poles_on_floor()
        load(c, t)
        g = assert_ground(c, t, gr.Params(15.0, 0.05, 0.2, 0.2, 10), "poles")
        assert_same(c.dense_segment_above_ground(0.15), gr.segment_above_ground(t.keys, t.cent, 0.1, g, 0.15), "above")
        t, g, pts, h = cloud_case()
        load(c, t)
        assert_ground(c, t, gr.Params(15.0, 0.05, 0.2, 0.2, 5), "cloud case")
        for hh in (h, 0.15):
            lab, ng = c.dense_ground_cloud(pts, IDENTITY, 2, hh)
            want = gr.ground_cloud(t, g, pts, IDENTITY, 2, hh)
            assert np.array_equal(lab, want[0]) and np.array_equal(ng.view(np.uint32), want[1].view(np.uint32))
    finally:
        c.close()


@pytest.mark.parametrize("leaf", [0.1, 0.2, 0.4])
def test_built_targets(build_libs, scene, leaf):
    """Targets built from HDL-64E map sweeps: the patches, the segmentation above the ground at 1.5, 2 and 4 leaves,
    the ground of sweeps at held-out poses; then the target saved and loaded back."""
    from loam_velodyne_b200 import synth
    c, ref = map_ctx(scene, synth.Lidar.hdl64(512), leaf)
    try:
        c.dense_target_build(None, 2, (0.0, 0.0, 0.0))
        cent, _, nrm = c.dense_export_normals(None, 2, (0.0, 0.0, 0.0))
        t = ar.Target(leaf, ref.keys, cent, nrm)
        prm = gr.Params(15.0, 0.05, float(np.float32(2 * leaf)), float(np.float32(1.5 * leaf)), 50)
        g = assert_ground(c, t, prm, f"leaf {leaf}")
        assert g.sum() > 1000
        for mult in (1.5, 2.0, 4.0):
            tol = float(np.float32(mult * leaf))
            assert_same(c.dense_segment_above_ground(tol, 2), gr.segment_above_ground(t.keys, t.cent, leaf, g, tol, 2),
                        f"leaf {leaf} above {tol}")
        pts = ar.static_sweep(scene, synth.Lidar.hdl64(512), HELD_OUT[1].astype(np.float64), seed=81)[0]
        lab, ng = c.dense_ground_cloud(pts, HELD_OUT[1], 1, 0.1)
        want = gr.ground_cloud(t, g, pts, HELD_OUT[1], 1, 0.1)
        assert np.array_equal(lab, want[0]) and np.array_equal(ng, want[1]) and (lab == 1).sum() > 100
        c.dense_target_load(leaf, cent, nrm)
        with pytest.raises(api_error(), match="invalid call sequence"):
            c.dense_segment_above_ground(0.3)  # the load dropped the ground
        t2 = ar.loaded_target(leaf, cent, nrm)
        assert_ground(c, t2, prm, f"leaf {leaf} reloaded")
    finally:
        c.close()


def api_error():
    from loam_velodyne_b200 import api
    return api.LoamB200Error


def test_floor_twice_and_identity(build_libs):
    """The 120 000-voxel floor: every voxel a candidate and one patch (every hook on one root), twice; with a min_size
    above the target nothing is ground and the segmentation above it is dense_segment, bit for bit."""
    from loam_velodyne_b200 import api
    leaf = 0.1
    pts = ground_plane(leaf)
    t = ar.loaded_target(leaf, pts, np.tile(np.float32([0, 1, 0, 0]), (pts.shape[0], 1)))
    c = api.Ctx(0)
    try:
        load(c, t)
        prm = gr.Params(15.0, 0.05, 0.15, 0.1, 1)
        want = gr.dense_ground(t.keys, t.cent, t.nrm, leaf, prm)
        assert want[1]["size"].tolist() == [120000]
        for _ in range(2):
            assert_same(c.dense_ground(prm.ctypes()), want[:2], "floor")
        assert c.dense_segment_above_ground(0.15)[1]["size"].size == 0
        t = poles_on_floor()
        load(c, t)
        lab, _ = c.dense_ground(gr.Params(min_size=10**6).ctypes())
        assert (lab == -1).all()
        for tol in (0.1, 0.15, 0.3):
            assert_same(c.dense_segment_above_ground(tol, 2), c.dense_segment(tol, 2), f"identity {tol}")
    finally:
        c.close()


def test_cloud_from_host_and_device(build_libs, scene):
    """A sweep with NaNs from host and device memory, the device output fed straight into cloud_segment."""
    import torch
    from loam_velodyne_b200 import api, synth
    c, ref = map_ctx(scene, synth.Lidar.vlp16(), 0.2)
    try:
        c.dense_target_build(None, 2, (0.0, 0.0, 0.0))
        cent, _, nrm = c.dense_export_normals(None, 2, (0.0, 0.0, 0.0))
        t = ar.Target(0.2, ref.keys, cent, nrm)
        g = gr.dense_ground(t.keys, t.cent, t.nrm, 0.2, gr.Params())[2]
        c.dense_ground()
        pts = ar.static_sweep(scene, synth.Lidar.hdl64(1024), HELD_OUT[0].astype(np.float64), seed=90)[0]
        pts[::97, 1] = np.nan
        pts[5::211, 0] = np.inf
        want = gr.ground_cloud(t, g, pts, HELD_OUT[0], 2, 0.15)
        lab, ng = c.dense_ground_cloud(pts, HELD_OUT[0], 2, 0.15)
        assert np.array_equal(lab, want[0]) and np.array_equal(ng, want[1])
        assert (lab == 1).sum() > 1000 and (lab == 0).sum() > 1000 and (lab == -1).sum() > 100
        dev = torch.from_numpy(pts).cuda()
        out = torch.full_like(dev, -7.0)
        lab_d, k = c.dense_ground_cloud(dev.data_ptr(), HELD_OUT[0], 2, 0.15, on_device=True, n=pts.shape[0],
                                        out=out.data_ptr())
        assert np.array_equal(lab_d, want[0]) and k == want[1].shape[0]
        assert np.array_equal(out[:k].cpu().numpy(), want[1])
        assert_same(c.segment_cloud(out.data_ptr(), 0.5, 3, on_device=True, n=k), sr.cloud_segment(want[1], 0.5, 3),
                    "objects")
    finally:
        c.close()


def test_errors_capacity_launches_and_products(build_libs, scene):
    from loam_velodyne_b200 import api, synth
    leaf = 0.2
    E = api.LoamB200Error
    c = api.Ctx(0)
    try:
        with pytest.raises(E, match="invalid call sequence"):
            c.dense_ground()  # no target
    finally:
        c.close()
    c, ref = map_ctx(scene, synth.Lidar.vlp16(), leaf)
    try:
        n = c.dense_target_build(None, 2, (0.0, 0.0, 0.0))
        with pytest.raises(E, match="invalid call sequence"):
            c.dense_segment_above_ground(0.3)  # no ground yet
        sweep = ar.static_sweep(scene, synth.Lidar.vlp16(), HELD_OUT[0].astype(np.float64), seed=70)[0]
        with pytest.raises(E, match="invalid call sequence"):
            c.dense_ground_cloud(sweep, HELD_OUT[0])
        lo, dims = api.voxel_box((-4.0, -2.0, -4.0), (4.0, 1.5, 4.0), leaf)
        rays = api.lidar_rays([-10.0, 0.0, 10.0], 256)
        c.dense_place_build(np.float32([[0.0, 0.0, 4.0 * k] for k in range(8)]), rays)

        def products():
            r = c.dense_raycast(rays, HELD_OUT[0], 0.0, 50.0)
            d = c.dense_distance_field(lo, dims, 1.0)
            s = c.dense_snapshot()
            q = c.dense_place_query(sweep)
            lab, seg = c.dense_segment(0.5)
            return [r[0], r[1], d[0], d[1], lab, seg["size"], seg["centroid"]] + [np.asarray(v) for v in s.values()] + \
                [np.asarray([(m["candidate"], m["shift"], m["dist"]) for m in q])]

        before = products()
        prm = gr.Params(15.0, 0.05, 0.4, 0.3, 20)
        for bad in (gr.Params(tol=np.nan), gr.Params(tol=0.0), gr.Params(max_step=-1.0), gr.Params(max_step=np.inf),
                    gr.Params(tol=float(np.float32(4 * leaf)) * 1.001), gr.Params(max_slope_deg=90.0),
                    gr.Params(max_slope_deg=-1.0), gr.Params(max_curvature=np.nan), gr.Params(max_curvature=-0.1),
                    gr.Params(min_size=0)):
            with pytest.raises(E, match="invalid argument"):
                c.dense_ground(bad.ctypes())
        with pytest.raises(E, match="invalid call sequence"):
            c.dense_segment_above_ground(0.3)  # the refusals stored nothing
        t = ar.Target(leaf, ref.keys, *c.dense_export_normals(None, 2, (0.0, 0.0, 0.0))[::2])
        want = gr.dense_ground(t.keys, t.cent, t.nrm, leaf, prm)
        c.profile(True)
        l0 = c.launch_count()
        got = c.dense_ground(prm.ctypes())
        ground_launches = c.launch_count() - l0
        prof = c.profile_get()
        assert prof["dense"][1] == ground_launches and sum(v[1] for k, v in prof.items() if k != "dense") == 0
        assert_same(got, want[:2], "first")
        K = got[1]["size"].size
        assert K > 3
        seg = (api.Segment * 4)()
        k = C.c_int(0)
        p = prm.ctypes()
        # capacity: the count comes back, the ground is stored all the same
        assert c.L.loam_b200_dense_ground(c.h, C.byref(p), None, seg, 3, C.byref(k)) == -5 and k.value == K
        assert c.L.loam_b200_dense_ground(c.h, C.byref(p), None, None, 1, C.byref(k)) == -1
        assert c.L.loam_b200_dense_ground(c.h, None, None, seg, 4, C.byref(k)) == -1
        assert c.L.loam_b200_dense_ground(c.h, C.byref(p), None, seg, 4, None) == -1
        above = gr.segment_above_ground(t.keys, t.cent, leaf, want[2], 0.5, 3)
        l0 = c.launch_count()
        assert_same(c.dense_segment_above_ground(0.5, 3), above, "above after ERR_CAPACITY")
        above_launches = c.launch_count() - l0
        for tol in (float(np.float32(4 * leaf)) * 1.001, np.nan):
            with pytest.raises(E, match="invalid argument"):
                c.dense_segment_above_ground(tol)
        for args in ((HELD_OUT[0], 0), (HELD_OUT[0], 4), (HELD_OUT[0], 1, -0.1), (HELD_OUT[0], 1, np.inf),
                     (np.float32([np.nan, 0, 0, 0, 0, 0]),)):
            with pytest.raises(E, match="invalid argument"):
                c.dense_ground_cloud(sweep, *args)
        l0 = c.launch_count()
        c.dense_ground_cloud(sweep, HELD_OUT[0])
        cloud_launches = c.launch_count() - l0
        assert cloud_launches == 4
        l0 = c.launch_count()
        c.dense_ground_cloud(np.zeros((0, 4), np.float32), HELD_OUT[0])
        assert c.launch_count() == l0
        # the launch count follows the target size and the candidate / entry counts only
        seg_of = {}
        c2 = api.Ctx(0)
        try:
            for m in (int((want[2]).sum()), n - int(want[2].sum()), int(gr.candidates(t.nrm, prm).sum())):
                plane = ground_plane(leaf)[:m]
                c2.dense_target_load(leaf, plane, np.tile(np.float32([0, 0, 1, 0]), (m, 1)))
                l0 = c2.launch_count()
                c2.dense_segment(0.5)
                seg_of[m] = c2.launch_count() - l0
        finally:
            c2.close()
        cand = int(gr.candidates(t.nrm, prm).sum())
        assert ground_launches == 5 + seg_of[cand]
        assert above_launches == 4 + seg_of[n - int(want[2].sum())]
        after = products()
        for a, b in zip(before, after):
            assert np.array_equal(np.atleast_1d(a).view(np.uint8), np.atleast_1d(b).view(np.uint8))
        # a rebuild drops the ground
        c.dense_target_build(None, 2, (0.0, 0.0, 0.0))
        with pytest.raises(E, match="invalid call sequence"):
            c.dense_segment_above_ground(0.5)
    finally:
        c.close()


def test_drop_in_equals_ctx(build_libs, scene):
    from loam_velodyne_b200 import api, synth
    c, _ = map_ctx(scene, synth.Lidar.vlp16(), 0.1)
    try:
        c.dense_target_build(None, 2, (0.0, 0.0, 0.0))
        cent, _, nrm = c.dense_export_normals(None, 2, (0.0, 0.0, 0.0))
        m = api.LaserMapping(0.1, 10)
        m.load_dense_target(0.1, cent, nrm)
        c.dense_target_load(0.1, cent, nrm)
        with pytest.raises(api.LoamB200Error):
            m.segment_dense_target_above_ground(0.2)
        assert_same(m.ground_dense_target(), c.dense_ground(), "ground")
        for tol, mn, mx in ((0.15, 1, None), (0.3, 5, 2000)):
            assert_same(m.segment_dense_target_above_ground(tol, mn, mx), c.dense_segment_above_ground(tol, mn, mx),
                        f"above {tol}")
        pts = ar.static_sweep(scene, synth.Lidar.vlp16(), HELD_OUT[2].astype(np.float64), seed=91)[0]
        pts[::50, 2] = np.nan
        lab, ng = c.dense_ground_cloud(pts, HELD_OUT[2], 1, 0.1)
        g, ng2 = m.split_ground(pts, HELD_OUT[2], 1, 0.1)
        assert np.array_equal(g, pts[lab == 1]) and np.array_equal(ng2, ng) and g.shape[0] > 100
    finally:
        c.close()
