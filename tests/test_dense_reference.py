"""The numpy restatement of the whole-run voxel map (tests/dense_reference.py) against the checker's pcl::VoxelGrid on
single clouds: same voxels in the same order, centroids within a few ulp (VoxelGrid sums in fp32, the map in fp64).
The GPU tests (test_dense_map.py) then trust the restatement bit for bit."""
import math

import numpy as np
import pytest

import dense_reference as dr

LEAVES = [0.05, 0.1, 0.2, 0.4]


def registered(pts, yaw, t):
    """A sweep moved into a map frame (rotation about y, translation) so that coordinates of both signs occur."""
    c, s = np.float32(math.cos(yaw)), np.float32(math.sin(yaw))
    p = np.array(pts, np.float32, copy=True)
    x, z = p[:, 0].copy(), p[:, 2].copy()
    p[:, 0] = c * x + s * z + np.float32(t[0])
    p[:, 1] = p[:, 1] + np.float32(t[1])
    p[:, 2] = -s * x + c * z + np.float32(t[2])
    return p


@pytest.fixture(scope="module")
def clouds(scene):
    from loam_velodyne_b200 import synth
    out = {}
    for name, lidar in (("vlp16", synth.Lidar.vlp16()), ("hdl64", synth.Lidar.hdl64())):
        pts, _ = synth.make_sweep(scene, lidar, 3, yaw_rate=math.radians(5.0))
        out[name] = registered(pts, 0.7, (-31.3, 1.7, 12.9))
    return out


def fits_voxel_grid(pts, leaf):
    """pcl::VoxelGrid keeps a cloud unfiltered when its voxel count overflows int32; crop the cloud until it fits."""
    r = 200.0
    while True:
        p = pts[np.all(np.abs(pts[:, :3]) < r, axis=1)]
        inv = np.float32(1.0) / np.float32(leaf)
        ext = [(np.floor(p[:, a].max() * inv) - np.floor(p[:, a].min() * inv) + 1) for a in range(3)]
        if float(ext[0]) * float(ext[1]) * float(ext[2]) < 2**31 - 1:
            return p
        r *= 0.8


def assert_close_to_voxel_grid(ref_c, pcl_c, max_ulp):
    assert ref_c.shape == pcl_c.shape
    sp = np.spacing(np.maximum(np.abs(ref_c), np.abs(pcl_c)).astype(np.float32))
    ulp = np.abs(ref_c.astype(np.float64) - pcl_c.astype(np.float64)) / sp
    assert ulp.max() <= max_ulp, f"max {ulp.max()} ulp"


@pytest.mark.parametrize("leaf", LEAVES)
@pytest.mark.parametrize("lidar", ["vlp16", "hdl64"])
def test_restatement_matches_voxel_grid(checker, clouds, lidar, leaf):
    pts = fits_voxel_grid(clouds[lidar], leaf)
    ref = dr.DenseMapRef(leaf)
    ref.insert(pts)
    c, n = ref.export()
    assert ref.stats() == {"voxels": c.shape[0], "skipped": 0, "dropped": 0}
    assert int(n.sum()) == pts.shape[0]
    pcl = checker.voxel_grid(pts, leaf)
    # same voxels in the same order: every VoxelGrid centroid is the restatement's of the same rank
    assert_close_to_voxel_grid(c, pcl, 16)
    assert c.shape[0] > 1000


def test_restatement_order_is_voxel_grid_order(clouds):
    """Ascending keys = z-major, then y, then x: the order of VoxelGrid's linear index."""
    k = np.unique(dr.voxel_keys(clouds["vlp16"], 0.2))
    v = dr.key_voxel(k)
    lex = np.lexsort((v[:, 0], v[:, 1], v[:, 2]))
    assert np.array_equal(lex, np.arange(k.size))


@pytest.mark.parametrize("leaf", LEAVES)
def test_key_edges_match_voxel_grid(checker, leaf):
    pts = dr.key_edge_cloud(leaf)
    k = dr.voxel_keys(pts, leaf)
    near = (k != dr.EMPTY) & np.all(np.abs(pts[:, :3]) < 100.0, axis=1)
    ref = dr.DenseMapRef(leaf)
    ref.insert(pts[near])
    c, _ = ref.export()
    assert_close_to_voxel_grid(c, checker.voxel_grid(pts[near], leaf), 4)


@pytest.mark.parametrize("leaf", LEAVES)
def test_key_edges(leaf):
    leaf32 = np.float32(leaf)
    inv = np.float32(1.0) / leaf32
    pts = dr.key_edge_cloud(leaf)
    k = dr.voxel_keys(pts, leaf)
    v = dr.key_voxel(k[k != dr.EMPTY])
    # a key is the voxel floorf(c * inv) of every axis, as VoxelGrid computes it
    f = np.floor(pts[k != dr.EMPTY, :3] * inv).astype(np.int64)
    assert np.array_equal(v, f)
    # faces land in voxel m, the float below them in m - 1
    for m in (0, 1, 3, -1, -3, 17, -17):
        assert m in v[:, 0] and m - 1 in v[:, 0]
    # -0.0 and tiny negatives: voxel 0 and -1
    assert dr.voxel_keys(np.array([[-0.0, -0.0, -0.0, 0]], np.float32), leaf)[0] == dr.voxel_keys(
        np.zeros((1, 4), np.float32), leaf)[0]
    assert tuple(dr.key_voxel(dr.voxel_keys(np.array([[-1e-30, 1e-30, -1e-30, 0]], np.float32), leaf))[0]) == (-1, 0, -1)
    # the range: -2^20 <= v < 2^20 on every axis, compared in float
    lo = np.float32(-dr.HALF) * leaf32
    assert np.floor(lo * inv) >= -dr.LIM
    assert dr.voxel_keys(np.array([[lo, 0, 0, 0]], np.float32), leaf)[0] != dr.EMPTY
    below = np.nextafter(lo, np.float32(-np.inf))
    while np.floor(below * inv) >= -dr.LIM:
        below = np.nextafter(below, np.float32(-np.inf))
    assert dr.voxel_keys(np.array([[0, 0, below, 0]], np.float32), leaf)[0] == dr.EMPTY
    hi = np.float32(dr.HALF) * leaf32
    while np.floor(hi * inv) < dr.LIM:
        hi = np.nextafter(hi, np.float32(np.inf))
    top = np.nextafter(hi, np.float32(-np.inf))
    assert dr.voxel_keys(np.array([[0, hi, 0, 0]], np.float32), leaf)[0] == dr.EMPTY
    kt = dr.voxel_keys(np.array([[top, top, top, 0]], np.float32), leaf)[0]
    assert tuple(dr.key_voxel([kt])[0]) == (dr.HALF - 1,) * 3
    assert kt < np.uint64(1 << 63)
    # NaN / inf on any axis: skipped
    bad = ~np.all(np.isfinite(pts[:, :3]), axis=1)
    assert bad.sum() == 9 and np.all(k[bad] == dr.EMPTY)
    ref = dr.DenseMapRef(leaf)
    ref.insert(pts)
    assert ref.stats()["skipped"] == int((k == dr.EMPTY).sum()) >= 9 + 6


def test_sequential_sums_differ_from_pairwise():
    """The restatement really sums sequentially: on values where pairwise summation rounds differently it keeps the
    sequential result, for short runs and for the long-run path alike."""
    rng = np.random.RandomState(5)
    for n in (40, dr.LONG_RUN + 50):
        x = (rng.uniform(-1, 1, n) * 10.0 ** rng.randint(-6, 7, n)).astype(np.float32)
        pts = np.stack([np.full(n, 0.01, np.float32)] * 3 + [x], axis=1)
        _, _, P, _ = dr.sweep_partials(pts, 1.0)
        seq = 0.0
        for v in x.astype(np.float64):
            seq += v
        assert P[0, 3] == seq


def test_cap_admits_in_key_order():
    pts = np.array([[x, 0.5, 0.5, 1.0] for x in (9.5, 0.5, 4.5, 2.5, 0.6, 7.5)], np.float32)
    ref = dr.DenseMapRef(1.0, max_voxels=3)
    ref.insert(pts)
    c, n = ref.export()
    assert np.array_equal(c[:, 0], np.float32([(0.5 + 0.6) / 2, 2.5, 4.5])) and list(n) == [2, 1, 1]
    assert ref.stats() == {"voxels": 3, "skipped": 0, "dropped": 2}
    ref.insert(np.array([[2.5, 0.5, 0.5, 3.0], [1.5, 0.5, 0.5, 0.0]], np.float32))
    c, n = ref.export()
    assert list(n) == [2, 2, 1] and c[1, 3] == 2.0 and ref.stats()["dropped"] == 3
