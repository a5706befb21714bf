"""The numpy restatement of the alignment against the whole-run voxel map (tests/align_reference.py), on the CPU: its
vectorised search against a brute-force scan of every target voxel, the hand-made edge cases against deliberately
wrong restatements, the export -> load round trip, pose recovery on static sweeps, and a degenerate one-plane target."""

import numpy as np
import pytest

import align_reference as ar
import dense_reference as dr


@pytest.fixture(scope="module")
def drv(build_libs):
    from oracle import pydriver
    return pydriver.best()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same(a, b):
    """Two iterate() results are equal bit for bit (NaN equal to NaN)."""
    return (np.array_equal(bits(a[0]), bits(b[0])) and np.array_equal(a[1], b[1]) and
            np.array_equal(bits(a[2]), bits(b[2])) and np.array_equal(a[3], b[3]))


# map sweeps and held-out sweeps of the recovery tests: (rot_x, rot_y, rot_z, x, y, z)
MAP_TWISTS = [np.array([0.0, 0.1 * k, 0.0, 0.5 * k, 0.0, 4.0 * k]) for k in range(4)]
HELD_OUT = [np.array([0.01, 0.15 * h + 0.05, -0.01, 0.3 * h, 0.0, 2.0 + 4.0 * h], np.float32) for h in range(3)]
# recovered error bars: the worst of the restatement's runs below was 2.7 mm and 0.061 deg (VLP-16, leaf 0.2)
BAR_M, BAR_DEG = 0.01, 0.1


def lidars():
    from loam_velodyne_b200 import synth
    return {"vlp16": synth.Lidar.vlp16(900), "hdl64": synth.Lidar.hdl64(512)}


def static_map(scene, lidar, leaf):
    ref = dr.DenseMapRef(leaf)
    for k, tw in enumerate(MAP_TWISTS):
        ref.insert(ar.static_sweep(scene, lidar, tw, seed=k)[1])
    return ref


def coarse_to_fine(align_fn, pts, init):
    a, _ = align_fn(pts, init, 3, 30)
    return align_fn(pts, a, 1, 30)


def test_search_matches_brute_force(scene, drv):
    """The box walk finds what a scan of every target voxel finds (the box contains the gate ball), with NaN normals
    present, at every radius; points are perturbed from a held-out pose so that many have no correspondence."""
    lidar = lidars()["hdl64"]
    ref = static_map(scene, lidar, 0.2)
    tgt = ar.built_target(ref, 1, (0.0, 0.0, 0.0), drv)
    assert np.isnan(tgt.nrm[:, 0]).sum() > 100
    pts = ar.static_sweep(scene, lidar, HELD_OUT[1].astype(np.float64), seed=50)[0][::11]
    import map_reference as mr
    q = mr.Pose(HELD_OUT[1] + np.array([0.01, -0.02, 0.0, 0.2, -0.1, 0.15], np.float32)).to_map(pts)
    q[::97, 0] = np.nan
    for radius in (1, 2, 3):
        fast, slow = ar.search(tgt, q, radius), ar.search_brute(tgt, q, radius)
        assert np.array_equal(fast, slow), f"radius {radius}: {int((fast != slow).sum())} of {q.shape[0]} differ"
        assert 0.2 * q.shape[0] < (fast >= 0).sum() < q.shape[0]


@pytest.mark.parametrize("name", list(ar.edge_cases()))
def test_edge_cases(name):
    cent, nrm, pts, twist, radius, variants = ar.edge_cases()[name]
    tgt = ar.loaded_target(ar.EDGE_LEAF, cent, nrm)
    right = ar.iterate(tgt, pts, twist, radius)
    match = right[1]
    expect = {"tie": [0], "gate": [-1], "no_normal": [1], "key_range": [-1, 0], "sensor_range": [0],
              "non_finite": [-1, -1, -1], "empty": [-1]}[name]
    assert match.tolist() == expect
    if variants is None:
        assert not right[0].any() and not right[2].any()
        return
    for v in variants:
        assert not same(right, ar.iterate(tgt, pts, twist, radius, **v)), f"{name}: {v} changes nothing"
    assert same(right, ar.iterate(tgt, pts, twist, radius, wrap=True)) or name != "key_range"


def test_round_trip_and_load_errors(scene, drv):
    """An exported centroid's voxel is its own voxel, so export -> load gives back the built target exactly; a
    duplicate voxel and an out-of-range or non-finite centroid are refused."""
    ref = static_map(scene, lidars()["vlp16"], 0.1)
    built = ar.built_target(ref, 2, (1.0, 2.0, 3.0), drv)
    loaded = ar.loaded_target(0.1, built.cent[::-1], built.nrm[::-1])
    assert np.array_equal(loaded.keys, built.keys)
    assert np.array_equal(bits(loaded.cent), bits(built.cent)) and np.array_equal(bits(loaded.nrm), bits(built.nrm))
    dup = np.concatenate([built.cent, built.cent[5:6] + np.float32(1e-3)])
    with pytest.raises(ValueError, match="same voxel"):
        ar.loaded_target(0.1, dup, np.concatenate([built.nrm, built.nrm[5:6]]))
    for bad in (np.nan, np.inf, 2.0e6):
        c = built.cent.copy()
        c[7, 1] = bad
        with pytest.raises(ValueError, match="key range"):
            ar.loaded_target(0.1, c, built.nrm)


@pytest.mark.parametrize("leaf", [0.1, 0.2])
@pytest.mark.parametrize("sensor", ["vlp16", "hdl64"])
def test_pose_recovery(scene, drv, sensor, leaf):
    """Map from four static sweeps, align held-out sweeps from ~0.3 m / 2 deg off, radius 3 then 1."""
    lidar = lidars()[sensor]
    tgt = ar.built_target(static_map(scene, lidar, leaf), 2, (0.0, 0.0, 0.0), drv)
    for h in (0, 2):
        truth = HELD_OUT[h]
        pts = ar.static_sweep(scene, lidar, truth.astype(np.float64), seed=100 + h)[0]
        init = (truth + ar.perturbations(h, 1)[0]).astype(np.float32)
        got, info = coarse_to_fine(lambda p, t, r, it: ar.align(tgt, p, t, r, it), pts, init)
        e_m, e_deg = ar.twist_error(got, truth)
        assert info["converged"] and e_m <= BAR_M and e_deg <= BAR_DEG, (sensor, leaf, h, e_m, e_deg, info)
        assert info["n_selected"] > 0.1 * pts.shape[0] and info["rms"] < 0.02


def test_one_plane_is_degenerate(drv):
    cent, nrm, pts = ar.plane_case()
    tgt = ar.loaded_target(ar.EDGE_LEAF, cent, nrm)
    init = np.array([0.01, 0.0, -0.01, 0.0, 0.05, 0.0], np.float32)
    got, info = ar.align(tgt, pts, init, 1, 10, drv=drv)
    assert info["degenerate"] and info["n_selected"] > 1000
    assert np.abs(got[[1, 3, 5]] - init[[1, 3, 5]]).max() < 1e-3  # the unobservable directions barely move
    assert ar.align(tgt, pts[:0], init, 1, 10)[1]["iterations"] == 0
    assert not ar.align(ar.Target(0.5, [], [], []), pts, init, 1, 10)[1]["converged"]
