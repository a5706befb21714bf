"""The plain reference of the mapping stage's bookkeeping (tests/map_reference.py) against the checker's own
BasicLaserMapping, sweep by sweep.  With max_iter = 0 the checker optimises nothing, so its cube clouds follow from
its pose (_transformTobeMapped), its stacks and the bookkeeping this reference restates; the GPU map tests
(test_map_stage.py) then trust the reference bit for bit."""
import math

import numpy as np

import map_reference as mr

# (rot_x, rot_y, rot_z, x, y, z) of successive sweeps: yaw beyond 1 rad, a sensor next to a cube corner, runs far
# enough along -x / +x to roll the grid by +1 and then by -2, a position on the negative side of x = -75
SUMS = [
    (0.01, 1.3, -0.02, 0.3, 0.1, 0.2),
    (-0.02, 2.4, 0.03, 24.9, 0.5, 24.8),
    (0.0, -1.1, 0.0, -74.9, 0.2, -25.1),
    (0.03, 3.0, -0.01, -380.0, 1.0, 10.0),
    (0.0, -2.9, 0.02, 380.0, -1.0, -30.0),
    (0.0, 0.4, 0.0, -5.0, 0.0, 3.0),
]


def far_points(n, seed):
    """Sparse points over the whole cube grid and beyond it (cubes that roll out, points the seed drops)."""
    rng = np.random.RandomState(seed)
    p = np.zeros((n, 4), np.float32)
    p[:, 0] = rng.uniform(-560, 560, n)
    p[:, 1] = rng.uniform(-300, 300, n)
    p[:, 2] = rng.uniform(-560, 560, n)
    p[:, 3] = rng.uniform(0, 16, n)
    return p


def test_reference_cube_bookkeeping_matches_checker(checker, scene, map_200k):
    from loam_velodyne_b200 import synth
    corner, surf = map_200k
    seed = (np.concatenate([corner, far_points(3000, 1)]), np.concatenate([surf, far_points(6000, 2)]))
    m = checker.mapping(0.1, 0)
    m.seed(*seed)
    maps = (mr.CubeMap(), mr.CubeMap())
    for cm, pts in zip(maps, seed):
        cm.add(pts)
    np.testing.assert_array_equal(maps[0].all_points(), m.cloud("corner_cubes"))
    np.testing.assert_array_equal(maps[1].all_points(), m.cloud("surf_cubes"))
    s = checker.scanreg()
    lidar = synth.Lidar.vlp16(n_az=900)
    rolls = set()
    for it, sum6 in enumerate(SUMS):
        pts, rs = synth.make_sweep(scene, lidar, it, yaw_rate=math.radians(5.0))
        s.process(pts, rs)
        m.set_inputs(s.cloud("less_sharp"), s.cloud("less_flat"), np.zeros((0, 4), np.float32))
        m.update_odometry(np.asarray(sum6, np.float32))
        assert m.process()
        # the window and the insertion both use _transformTobeMapped (aft only follows it when the optimisation ran)
        tobe = m.twist("tobe")
        stacks = (m.cloud("corner_stack_ds"), m.cloud("surf_stack_ds"))
        assert stacks[0].shape[0] > 50 and stacks[1].shape[0] > 50
        before = maps[0].cen
        _, from_map = mr.sweep_update(maps, (0.2, 0.4), tobe, tobe, stacks, checker.voxel_grid)
        rolls.add(tuple(int(a - b) for a, b in zip(maps[0].cen, before)))
        np.testing.assert_array_equal(from_map[0], m.cloud("corner_from_map"), err_msg=f"sweep {it}: corner from-map")
        np.testing.assert_array_equal(from_map[1], m.cloud("surf_from_map"), err_msg=f"sweep {it}: surface from-map")
        np.testing.assert_array_equal(maps[0].all_points(), m.cloud("corner_cubes"), err_msg=f"sweep {it}: corner cubes")
        np.testing.assert_array_equal(maps[1].all_points(), m.cloud("surf_cubes"), err_msg=f"sweep {it}: surface cubes")
    assert (1, 0, 0) in rolls and (-2, 0, 0) in rolls, rolls


def test_no_fp32_centroid_crosses_a_cube_face():
    """The GPU derives a point's cube from its coordinates; the reference keeps a point in the cube it was inserted into.
    The two agree as long as no voxel centroid rounds across a cube face.  Exhaustive for up to 512 points per voxel
    within 1024 ulps of every face of the grid, on both sides (the store_cell quirk puts x = -75, -125, ... into the
    lower cube); by monotonicity (map_reference.first_crossing) this covers every set of distinct values too."""
    cube_x = lambda x: mr.cube_ijk(np.stack([x, x * 0, x * 0, x * 0], axis=1), (10, 5, 10))[:, 0]
    for face in range(-525, 526, 50):
        for side in (-1, 1):
            assert mr.first_crossing(face, side, cube_x) is None, (face, side)
    # the same search does find crossings of ordinary voxel faces (test_map_stage.py::test_map_update_edges uses them)
    for leaf in (0.2, 0.4):
        inv = np.float32(1.0) / np.float32(leaf)
        k = int(np.floor(np.float32(-53.2) * inv))
        hit = mr.first_crossing(mr.voxel_face(k, leaf), -1, lambda x: np.floor(x * inv).astype(np.int64))
        assert hit is not None, leaf


def test_libm_sincos_in_poses():
    """Pose structs carry glibc sinf / cosf of the float angle, as loam::Angle caches them."""
    from loam_velodyne_b200 import api
    import ctypes
    import ctypes.util
    libm = ctypes.CDLL(ctypes.util.find_library("m"))
    libm.sinf.restype = libm.cosf.restype = ctypes.c_float
    libm.sinf.argtypes = libm.cosf.argtypes = [ctypes.c_float]
    rng = np.random.RandomState(4)
    ang = rng.uniform(-3.2, 3.2, 200).astype(np.float32)
    for a in ang:
        p = api.make_pose((a, -a, a * 0.5, 1, 2, 3))
        for i, v in enumerate((a, -a, np.float32(a * np.float32(0.5)))):
            assert np.float32(p.sin_[i]) == np.float32(libm.sinf(float(v)))
            assert np.float32(p.cos_[i]) == np.float32(libm.cosf(float(v)))
    # small angles (the pre-existing tests' poses) give numpy's values too
    for a in np.linspace(-0.05, 0.05, 101).astype(np.float32):
        s, c = api.sincos_f32(a)
        assert s == np.sin(a, dtype=np.float32) and c == np.cos(a, dtype=np.float32)
