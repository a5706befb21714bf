"""Carve mode restated in numpy (tests/carve_reference.py), on the CPU: the walk against a slab test over every stored
voxel, the hand-made cases against deliberately wrong restatements, and the trail of a moving box against the static
street scene with ground-truth poses over a sweep of margins, beside the range-image pass."""
import numpy as np
import pytest

import carve_reference as cr
import dense_reference as dr
import visibility_reference as vr
from test_visibility_reference import EXPECTED as RANGE_IMAGE_EXPECTED


def random_map(seed, leaf, m=400):
    rng = np.random.RandomState(seed)
    vox = np.unique(rng.randint(-6, 6, size=(m, 3)), axis=0)
    pts = ((vox + rng.uniform(0.05, 0.95, vox.shape)) * leaf).astype(np.float32)
    return np.concatenate([pts, np.ones((pts.shape[0], 1), np.float32)], axis=1)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_walk_matches_slab(seed):
    """The carved voxels of each ray are the stored voxels whose slab segment [max(t_near, 0), t_far] has positive
    length and ends at or before T = min(r - margin, max_range), for random origins and points; rays that pass within
    1e-9 m of a voxel edge or whose T lies within 1e-9 of a voxel's exit are excluded."""
    leaf = 0.3
    ref = vr.VisibilityMapRef(leaf)
    ref.insert(random_map(seed, leaf))
    keys = ref.keys
    rng = np.random.RandomState(100 + seed)
    n_carved = n_rays = 0
    for k in range(4):
        o = rng.uniform(-2.0, 2.0, 3).astype(np.float32)
        pts = np.concatenate([(o + rng.normal(scale=2.0, size=(200, 3))), np.ones((200, 1))], axis=1)
        pts = pts.astype(np.float32)
        for margin, mx in ((0.0, 100.0), (0.3, 100.0), (0.2, 1.5)):
            ray, j, t = cr.carve_walk(keys, leaf, pts, o, margin, mx)
            rows, en, tf, r = cr.slab(keys, leaf, pts, o)
            T = np.minimum(r - margin, mx)
            crossed = tf - en
            clear = ~((np.abs(crossed) < 1e-9) | (np.abs(tf - T[:, None]) < 1e-9)).any(axis=1)
            assert clear.mean() > 0.9
            want = (crossed > 0.0) & (tf <= T[:, None])
            got = np.zeros_like(want)
            at = np.searchsorted(rows, ray)
            got[at, j] = True
            assert np.array_equal(got[clear], want[clear]), (seed, k, margin, int((got[clear] != want[clear]).sum()))
            # a voxel is carved at most once per ray, in walk order (t_exit non-decreasing)
            assert np.unique(ray * keys.size + j).size == ray.size
            n_carved += int(want[clear].sum())
            n_rays += int(clear.sum())
    assert n_carved > 1000 and n_rays > 2000


@pytest.mark.parametrize("name", list(cr.edge_cases()))
def test_edge_cases(name):
    expect, variants = cr.edge_cases()[name][5:7]
    right = cr.run_case(name)
    assert right.misses.tolist() == expect
    assert cr.run_case(name, max_steps=4096).misses.tolist() == expect
    for v in variants:
        wrong = cr.run_case(name, **v)
        assert wrong.misses.tolist() != expect, f"{name}: {v} changes nothing"


def test_hits_unchanged_and_keys_in_k():
    """Carve mode changes only misses; K is the map's own voxel rule (a point on a voxel face belongs to the voxel
    above it)."""
    ref = cr.CarveMapRef(0.5, margin=0.0, max_range=50.0)
    ref.insert(np.array([[0.75, 0.25, 0.25, 1.0], [1.25, 0.25, 0.25, 1.0]], np.float32))
    # the ray ends exactly on the face x = 1.0, inside voxel 2 by floorf(1.0 * 2) = 2: voxel (1, 0, 0) is carved (its
    # exit 0.75 <= T = 0.75), voxel (2, 0, 0) is in K
    ref.observe(np.array([[1.0, 0.25, 0.25, 1.0]], np.float32), (0, 0, 0, 0.25, 0.25, 0.25))
    assert ref.misses.tolist() == [1, 0] and ref.hits.tolist() == [1, 1]
    assert dr.voxel_keys(np.array([[1.0, 0.25, 0.25, 1.0]], np.float32), 0.5)[0] == ref.keys[1]


# Measured with tests/carve_reference.py (24 sweeps, leaf 0.2 m, ratio 1, max_range 100 m, 10 m/s box 7 m ahead;
# trail and static as in test_visibility_reference), trail removed / static kept:
#   margin   VLP-16          HDL-64E
#   0.0      0.914 / 0.863   1.000 / 0.733
#   0.5      0.914 / 0.911   1.000 / 0.771
#   1.0      0.912 / 0.961   0.999 / 0.814
#   1.5      0.872 / 0.987   0.984 / 0.878
#   2.0      0.834 / 0.994   0.954 / 0.932   <- recommended (carve_reference.MARGIN)
#   2.5      0.788 / 0.996   0.925 / 0.966
#   3.0      0.735 / 0.996   0.890 / 0.982
# range image (1 deg x 2 deg, 1 m): VLP-16 0.961 / 0.947, HDL-64E 0.947 / 0.989.
MARGINS = (0.0, 0.5, 1.0, 1.5, 2.0, 2.5, 3.0)
EXPECTED = {"vlp16": (0.83, 0.99), "hdl64": (0.95, 0.93)}
RANGE_IMAGE = {"vlp16": (0.961, 0.947), "hdl64": (0.947, 0.989)}


@pytest.mark.parametrize("lidar", ["vlp16", "hdl64"])
def test_moving_box_trail(scene, lidar):
    from loam_velodyne_b200 import synth
    run = vr.moving_box_run(scene, getattr(synth.Lidar, lidar)(), 24)
    res = cr.margin_sweep(run, 0.2, MARGINS)
    for m in MARGINS:
        print(f"{lidar}: margin {m}: trail removed {res[m][0]:.4f}, static kept {res[m][1]:.4f}")
    removed, kept = res[cr.MARGIN]
    assert removed >= EXPECTED[lidar][0] and kept >= EXPECTED[lidar][1]
    # never worse than the range-image pass on both numbers at once
    ri = RANGE_IMAGE[lidar]
    assert removed > ri[0] or kept > ri[1]
    assert RANGE_IMAGE[lidar][0] >= RANGE_IMAGE_EXPECTED[lidar][0]
    # the margin trades removal for static kept: kept never falls as the margin grows
    kept_by_margin = [res[m][1] for m in MARGINS]
    assert kept_by_margin == sorted(kept_by_margin)


def test_margin_sweep_matches_full_runs(scene):
    """The sweep's prefix shortcut equals CarveMapRef run at each margin (a short VLP-16 run)."""
    from loam_velodyne_b200 import synth
    run = vr.moving_box_run(scene, synth.Lidar.vlp16(n_az=360), 6)
    res = cr.margin_sweep(run, 0.2, (0.5, 2.0), settle=1)
    trail, static = vr.trail_and_static(run, 0.2, 1)
    for m in (0.5, 2.0):
        ref = cr.CarveMapRef(0.2, margin=m)
        for pts, twist, _ in run:
            ref.sweep(pts, twist)
        assert vr.removal_rates(ref, trail, static, 1.0) == res[m]
