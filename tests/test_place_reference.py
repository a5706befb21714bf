"""The numpy restatement of the place descriptor and match (tests/place_reference.py), on the CPU: the sector rule
against plain atan2 binning and against the device's bisection, hand-made cases each changed by a deliberately wrong
restatement, and the yaw convention on a small restated target."""
import math

import numpy as np
import pytest

import align_reference as ar
import place_reference as pr
import raycast_reference as rr
from test_align_reference import lidars, static_map

P = pr.Params(rings=4, sectors=8, max_radius=8.0, height_offset=2.0)  # w = 2 m, D = 45 deg


@pytest.fixture(scope="module")
def drv(build_libs):
    from oracle import pydriver
    return pydriver.best()


def pts(rows):
    return np.array([list(r) + [0.0] * (4 - len(r)) for r in rows], np.float32).reshape(-1, 4)


def bisect(x, z, sectors):
    """The device's search: the count of boundaries past, by bisection over [1, sectors)."""
    c, s = pr.boundaries(sectors)
    hp = 0 if (x > 0.0 or (x == 0.0 and z > 0.0)) else 1
    lo, hi = 1, sectors
    while lo < hi:
        mid = (lo + hi) >> 1
        hk = 1 if 2 * mid >= sectors else 0
        if hp > hk or (hp == hk and x * c[mid] - z * s[mid] >= 0.0):
            lo = mid + 1
        else:
            hi = mid
    return lo - 1


@pytest.mark.parametrize("sectors", [1, 2, 7, 60, 720])
def test_sector_rule(sectors):
    """Away from wedge edges the rule is atan2 binning; everywhere its count equals the device's bisection."""
    rng = np.random.RandomState(sectors)
    p = rng.normal(size=(4000, 2)) * rng.choice([1e-3, 1.0, 50.0], size=(4000, 1))
    p = np.concatenate([p, [[0.0, 1.0], [0.0, -1.0], [1.0, 0.0], [-1.0, 0.0], [1e-30, -1.0], [-1e-30, 1.0]]])
    x, z = p[:, 0].astype(np.float32).astype(np.float64), p[:, 1].astype(np.float32).astype(np.float64)
    got = pr.sectors_of(x, z, sectors)
    d = pr.step(sectors)
    a = np.mod(np.arctan2(x, z), 2.0 * math.pi)
    off = np.abs(a / d - np.round(a / d)) * d
    far = (off > 1e-9) & (np.abs(a - 2.0 * math.pi) > 1e-9)
    assert far.sum() > 3900
    assert np.array_equal(got[far], pr.sectors_atan2(x, z, sectors)[far])
    assert all(bisect(x[i], z[i], sectors) == got[i] for i in range(x.size))
    assert got.min() >= 0 and got.max() <= sectors - 1


def on_boundary_point():
    """A float point on the 45-deg boundary with x * cos - z * sin == 0 exactly."""
    c, s = pr.boundaries(8)
    for v in np.arange(1.0, 7.0, 1.0 / 1024, dtype=np.float32):
        if float(v) * c[1] - float(v) * s[1] == 0.0:
            return float(v)
    raise AssertionError("no exact boundary point")


def cases():
    """{name: (points, check(descriptor) -> bool, variant)}"""
    b = on_boundary_point()
    out = {}
    out["wedge_boundary"] = (pts([(b, 1.0, b)]), lambda d: d[int(math.hypot(b, b) // 2.0), 1] == np.float32(3.0),
                             {"edge_gt": True})
    out["ring_boundary"] = (pts([(0.0, 1.0, 4.0)]), lambda d: d[2, 0] == np.float32(3.0), {"ring_ceil": True})
    out["max_radius"] = (pts([(0.0, 1.0, 8.0)]), lambda d: not d.any(), {"r_gt": True})
    out["zero_radius"] = (pts([(0.0, 5.0, 0.0)]), lambda d: not d.any(), {"keep_zero_r": True})
    out["non_finite"] = (pts([(np.nan, 1.0, 3.0), (1.0, np.inf, 3.0), (np.inf, 1.0, 3.0)]), lambda d: not d.any(),
                         {"nan_as_zero": True})
    out["value_not_positive"] = (pts([(0.0, -3.0, 3.0), (0.0, -2.0, 5.0)]), lambda d: not d.any(),
                                 {"signed_max": True})
    out["two_in_one_bin"] = (pts([(0.1, 1.0, 3.0), (0.2, -1.0, 3.5)]), lambda d: d[1, 0] == np.float32(3.0),
                             {"last_wins": True})
    return out


@pytest.mark.parametrize("name", list(cases()))
def test_descriptor_cases(name):
    p, check, variant = cases()[name]
    assert check(pr.descriptor(p, P)), name
    assert not np.array_equal(pr.descriptor(p, P, **variant), pr.descriptor(p, P)), name


def random_desc(rng, prm, empty_cols=()):
    d = rng.uniform(0.0, 10.0, (prm.rings, prm.sectors)).astype(np.float32)
    d[rng.uniform(size=d.shape) < 0.3] = 0.0
    for c in empty_cols:
        d[:, c] = 0.0
    return d


def test_distance_cases():
    rng = np.random.RandomState(4)
    q = random_desc(rng, P, empty_cols=(2,))
    d = random_desc(rng, P)
    # empty columns are skipped; with every column empty there is no distance
    assert not np.array_equal(pr.distances(q, d), pr.distances(q, d, no_skip=True))
    z = np.zeros_like(q)
    assert np.isinf(pr.distances(z, d)).all() and np.isinf(pr.distances(q, z)).all()
    assert not np.isinf(pr.distances(z, d, no_skip=True)).any()
    # a rolled descriptor is found at distance 0 at its shift: query column j is candidate column (j + s0)
    s0 = 3
    rolled = np.roll(d, -s0, axis=1)
    assert np.array_equal(rolled[:, 0], d[:, s0])
    dist, s = pr.best_shift(pr.distances(rolled, d))
    assert s == s0 and abs(dist) < 1e-15
    assert pr.best_shift(pr.distances(rolled, d, shift_sign=True))[1] == P.sectors - s0
    # shift ties go to the smaller shift; index ties to the smaller index
    flat = np.tile(rng.uniform(1.0, 2.0, (P.rings, 1)).astype(np.float32), (1, P.sectors))
    dist = pr.distances(flat, flat)
    assert (dist == dist[0]).all()
    assert pr.best_shift(dist)[1] == 0 and pr.best_shift(dist, tie_last=True)[1] == P.sectors - 1
    db = np.stack([d, rolled, d, z])
    bd, bs = pr.query(rolled, db)
    assert np.isinf(bd[3]) and bd[0] == bd[2]
    order = pr.top_m(bd, 3).tolist()
    assert sorted(order) == [0, 1, 2] and order.index(0) < order.index(2)
    assert pr.top_m(bd, 4).size == 3  # never one at +inf
    rev = pr.top_m(bd, 3, index_desc=True).tolist()
    assert rev.index(2) < rev.index(0)
    assert pr.yaw_of(30, 60) == np.float32(math.pi) and pr.yaw_of(31, 60) < 0 and pr.yaw_of(5, 60) > 0


def test_yaw_sign(scene, drv):
    """A static sweep at heading psi from a place recovers shift round(psi / D) against the place's rendered
    descriptor (the map side restated: dense_reference + raycast_reference)."""
    from loam_velodyne_b200 import api
    lidar = lidars()["vlp16"]
    ref = static_map(scene, lidar, 0.2)
    tgt = ar.built_target(ref, 2, (0.0, 0.0, 0.0), drv)
    prm = pr.Params(rings=10, sectors=36, max_radius=40.0, height_offset=2.0, max_range=40.0)
    place = np.array([0.75, 0.0, 6.0], np.float32)
    rays = api.lidar_rays(np.linspace(lidar.lower_deg, lidar.upper_deg, lidar.n_rings), 360)
    rng, _ = rr.cast(tgt, rays, np.concatenate([np.zeros(3, np.float32), place]), prm.min_range, prm.max_range)
    d = pr.descriptor(pr.rendered_points(rays, rng), prm)
    D = pr.step(prm.sectors)
    for s0 in (0, 4, 17, 31):
        psi = (s0 if 2 * s0 <= prm.sectors else s0 - prm.sectors) * D
        q = ar.static_sweep(scene, lidar, np.array([0.0, psi, 0.0, *place], np.float64), seed=s0)[0]
        dist, s = pr.best_shift(pr.distances(pr.descriptor(q, prm), d))
        assert s == s0, (s0, s, dist)
        assert abs(pr.yaw_of(s, prm.sectors) - psi) < 1e-6
