"""The visibility pass restated in numpy (tests/visibility_reference.py): hand-made geometry, and the trail of a moving
box against the static street scene with ground-truth poses at the recommended parameters."""
import math

import numpy as np
import pytest

import visibility_reference as vr

IDENTITY = (0.0, 0.0, 0.0, 0.0, 0.0, 0.0)
# recommended parameters (DESIGN.md "Visibility pass"): 1 deg x 2 deg pixels, 1 m margin, keep misses <= hits
H_RES, V_RES, MARGIN, RATIO = 1.0, 2.0, 1.0, 1.0


def cloud(*xyz):
    return np.array([[x, y, z, 1.0] for x, y, z in xyz], np.float32)


def wall(z, half=2.0, step=0.01):
    g = np.arange(-half, half + step / 2, step, dtype=np.float32)
    x, y = np.meshgrid(g, g)
    return np.stack([x.ravel(), y.ravel(), np.full(x.size, z, np.float32), np.ones(x.size, np.float32)], axis=1)


def one_pass(stored, seen, pose=IDENTITY, h=0.5, v=0.5, margin=0.2):
    ref = vr.VisibilityMapRef(0.1, h_res=h, v_res=v, margin=margin)
    ref.insert(stored)
    ref.observe(seen, pose)
    return ref


def test_wall_in_front_and_behind():
    ref = one_pass(cloud((0.05, 0.05, 5.05), (0.05, 0.05, 15.05), (10.05, 0.05, 5.05)), wall(10.0))
    c = ref.centroids()
    miss = dict(zip(map(tuple, np.round(c, 2).tolist()), ref.misses.tolist()))
    assert miss[(0.05, 0.05, 5.05)] == 1  # in front of the wall: seen through
    assert miss[(0.05, 0.05, 15.05)] == 0  # behind it: occluded
    assert miss[(10.05, 0.05, 5.05)] == 0  # its pixel has no return: no evidence
    assert ref.hits.tolist() == [1, 1, 1]
    # seen from a pose turned away (yaw pi) and moved, the wall is behind the sensor: no evidence at all
    ref = one_pass(cloud((0.05, 0.05, 5.05)), wall(10.0), pose=(0.0, math.pi, 0.0, 0.0, 0.0, 20.0))
    assert ref.misses.tolist() == [0]


def test_threshold_is_strict():
    """r = 5 exactly (a point on the optical axis); the image holds 5.5.  r + margin == 5.5: no miss; r + margin one
    double below 5.5: a miss."""
    stored, seen = cloud((0.0, 0.0, 5.0)), cloud((0.0, 0.0, 5.5))
    assert one_pass(stored, seen, margin=0.5).misses.tolist() == [0]
    below = float(np.nextafter(5.5, 0.0)) - 5.0  # exact: 5.0 + below == nextafter(5.5, 0)
    assert 5.0 + below == np.nextafter(5.5, 0.0)
    assert one_pass(stored, seen, margin=below).misses.tolist() == [1]


def test_row_clamped_at_plus_90():
    """Straight up is elevation +90 deg: floor(180 / v_res) = rows, clamped to the top row, where a return at 89.5 deg
    elevation (same azimuth) also lands."""
    e = math.radians(89.5)
    seen = cloud((0.0, 30.0 * math.sin(e), 30.0 * math.cos(e)))
    r, pix, _ = vr.pixels(np.array([[0.0, 10.0, 0.0]]), IDENTITY, 1.0, 1.0)
    assert pix[0] // 360 == 179
    assert one_pass(cloud((0.0, 10.0, 0.0)), seen, h=1.0, v=1.0).misses.tolist() == [1]


def test_azimuth_wraps_at_180():
    """Azimuth +180 deg (x = +0, z < 0) gives floor(360 / h_res) = cols -> column 0, where azimuth -179.9 deg lands."""
    a = math.radians(-179.9)
    seen = cloud((20.0 * math.sin(a), 0.0, 20.0 * math.cos(a)))
    r, pix, _ = vr.pixels(np.array([[0.0, 0.0, -5.0]]), IDENTITY, 1.0, 1.0)
    assert pix[0] % 360 == 0
    assert one_pass(cloud((0.0, 0.0, -5.0)), seen, h=1.0, v=1.0).misses.tolist() == [1]


def test_saturation():
    ref = one_pass(cloud((0.0, 0.0, 5.0)), cloud((0.0, 0.0, 9.0)))
    ref.misses[:] = vr.SAT - 1
    ref.hits[:] = vr.SAT - 1
    for _ in range(3):
        ref.observe(cloud((0.0, 0.0, 9.0)), IDENTITY)
        ref.insert(cloud((0.0, 0.0, 5.0)))
    assert ref.misses.tolist() == [vr.SAT] and ref.hits.tolist() == [vr.SAT]


def test_ratio_filter():
    ref = one_pass(cloud((0.0, 0.0, 5.0), (1.0, 0.0, 5.0)), cloud((0.0, 0.0, 9.0)))
    assert ref.misses.tolist() == [1, 0] and ref.hits.tolist() == [1, 1]
    assert ref.export_filtered(0.0)[0].shape[0] == 1
    assert ref.export_filtered(1.0)[0].shape[0] == 2
    c, n, h, m = ref.export_filtered()
    assert np.array_equal(c, ref.export()[0]) and np.array_equal(n, ref.export()[1])


# measured with these parameters (24 sweeps, leaf 0.2 m, 10 m/s box 7 m ahead; trail = voxels of box points only
# that the box left >= 6 sweeps before the end, static = voxels never holding a box point):
#   VLP-16: trail removed 0.961, static kept 0.947;  HDL-64E: trail removed 0.947, static kept 0.989.
# The end-to-end pipeline test (estimated poses) is held to the VLP-16 pair.
EXPECTED = {"vlp16": (0.95, 0.93), "hdl64": (0.94, 0.985)}


@pytest.mark.parametrize("lidar", ["vlp16", "hdl64"])
def test_moving_box_trail(scene, lidar):
    from loam_velodyne_b200 import synth
    run = vr.moving_box_run(scene, getattr(synth.Lidar, lidar)(), 24)
    trail, static = vr.trail_and_static(run, 0.2)
    assert len(trail) > 500 and len(static) > 50000
    ref = vr.VisibilityMapRef(0.2, h_res=H_RES, v_res=V_RES, margin=MARGIN)
    for pts, twist, _ in run:
        ref.sweep(pts, twist)
    removed, kept = vr.removal_rates(ref, trail, static, RATIO)
    print(f"{lidar}: trail removed {removed:.4f}, static kept {kept:.4f}")
    assert removed >= EXPECTED[lidar][0] and kept >= EXPECTED[lidar][1]
