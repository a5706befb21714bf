"""The numpy restatement of the distance field (tests/distance_reference.py) on the CPU: its exact transform against
scipy.ndimage.distance_transform_edt and a brute force, the padding claim against fields over much larger boxes, the
query's properties, and the hand-made cases each shown to catch a deliberately wrong restatement."""
import itertools
import math

import numpy as np
import pytest
from scipy import ndimage

import distance_reference as dist_ref


def scipy_sq(occ):
    return np.round(ndimage.distance_transform_edt(~occ) ** 2).astype(np.int64)


@pytest.mark.parametrize("shape,density,seed", [((17, 23, 19), 0.01, 1), ((9, 31, 12), 0.05, 2),
                                                ((40, 40, 40), 0.002, 3), ((6, 5, 50), 0.2, 4),
                                                ((1, 30, 30), 0.03, 5), ((30, 1, 30), 0.03, 6), ((30, 30, 1), 0.03, 7),
                                                ((1, 1, 64), 0.05, 8), ((64, 1, 1), 0.05, 9), ((25, 25, 25), 0.0005, 10)])
def test_against_scipy(shape, density, seed):
    rng = np.random.RandomState(seed)
    occ = rng.uniform(size=shape) < density
    occ.flat[rng.randint(occ.size)] = True  # at least one obstacle (scipy has no value without one)
    assert np.array_equal(dist_ref.edt_sq(occ), scipy_sq(occ))


def test_degenerate_grids():
    for shape in ((1, 1, 1), (1, 4, 1), (3, 3, 3), (2, 1, 7)):
        assert (dist_ref.edt_sq(np.ones(shape, bool)) == 0).all()
        assert (dist_ref.edt_sq(np.zeros(shape, bool)) == dist_ref.INF).all()
        one = np.zeros(shape, bool)
        one.flat[-1] = True
        assert np.array_equal(dist_ref.edt_sq(one), scipy_sq(one))


@pytest.mark.parametrize("seed", range(6))
def test_brute_force(seed):
    rng = np.random.RandomState(seed)
    shape = tuple(rng.randint(1, 7, 3))
    occ = rng.uniform(size=shape) < 0.15
    got = dist_ref.edt_sq(occ)
    sites = np.argwhere(occ)
    for idx in itertools.product(*(range(s) for s in shape)):
        want = ((sites - np.array(idx)) ** 2).sum(axis=1).min() if sites.size else dist_ref.INF
        assert got[idx] == want, (idx, got[idx], want)


def random_target(seed, n=300, span=40):
    rng = np.random.RandomState(seed)
    vox = np.unique(rng.randint(-span, span, (n, 3)), axis=0)
    return dist_ref.keys_of_voxels(vox), vox


# (leaf, max_distance): non-integer ratios and integer multiples (0.3 / 0.1 rounds to just below 3 in double)
RATIOS = [(0.1, 0.3), (0.1, 0.35), (0.2, 1.0), (0.25, 1.0), (0.5, 1.0), (0.4, 2.0), (0.1, 1.05), (0.3, 2.1)]


@pytest.mark.parametrize("leaf,md", RATIOS)
def test_padding_claim(leaf, md):
    """A box's field equals the same cells cut from the field over a box grown by 16 voxels per side (more than any
    pad here; its own pad only adds more), with the beyond cells alike; and every reported value equals the transform
    of the whole target, every beyond cell being truly beyond."""
    keys, vox = random_target(11, n=250, span=30)
    G = 16
    for lo, dims in (((-10, -7, -12), (14, 9, 20)), ((5, 5, 5), (6, 4, 3)), ((-40, -3, 20), (12, 6, 15))):
        assert dist_ref.pad_of(leaf, md) < G
        dist, sq = dist_ref.field(keys, leaf, lo, dims, md)
        bdist, bsq = dist_ref.field(keys, leaf, np.array(lo) - G, np.array(dims) + 2 * G, md)
        cut = (slice(G, G + dims[2]), slice(G, G + dims[1]), slice(G, G + dims[0]))
        assert np.array_equal(sq, bsq[cut])
        assert np.array_equal(dist.view(np.uint32), bdist[cut].view(np.uint32))
        # the whole target: a grid over every target voxel and the box
        wlo = np.minimum(vox.min(axis=0), lo)
        whi = np.maximum(vox.max(axis=0), np.array(lo) + np.array(dims) - 1)
        whole = dist_ref.edt_sq(dist_ref.occupancy(vox, wlo, whi - wlo + 1))
        o = np.array(lo) - wlo
        w = whole[o[2]:o[2] + dims[2], o[1]:o[1] + dims[1], o[0]:o[0] + dims[0]]
        inside = sq >= 0
        assert np.array_equal(sq[inside], w[inside])
        L = float(np.float32(leaf))
        assert (np.sqrt(w[~inside].astype(np.float64)) * L > float(np.float32(md))).all()


def test_field_values():
    keys, _ = random_target(3, n=120, span=12)
    dist, sq = dist_ref.field(keys, 0.2, (-14, -14, -14), (28, 28, 28), 1.5)
    assert (sq == 0).sum() == keys.size and (sq == -1).any() and (sq > 0).any()
    L = float(np.float32(0.2))
    ok = sq >= 0
    assert np.array_equal(dist[ok], (np.sqrt(sq[ok].astype(np.float64)) * L).astype(np.float32))
    assert np.isinf(dist[~ok]).all() and (dist[ok] <= np.float32(1.5)).all()


def test_empty_target():
    dist, sq = dist_ref.field(np.zeros(0, np.uint64), 0.1, (0, 0, 0), (4, 3, 2), 1.0)
    assert sq.shape == (2, 3, 4) and (sq == -1).all() and np.isinf(dist).all()


def wrong_variants():
    return {"beyond_ge": dict(beyond_ge=True), "ignore_outside": dict(ignore_outside=True)}


def test_wrong_restatements_are_caught():
    """Each deliberately wrong field restatement changes some hand-made case."""
    cases = dist_ref.edge_cases()
    for name, kw in wrong_variants().items():
        changed = []
        for case, (leaf, vox, lo, dims, md) in cases.items():
            keys = dist_ref.keys_of_voxels(vox)
            a = dist_ref.field(keys, leaf, lo, dims, md)[1]
            b = dist_ref.field(keys, leaf, lo, dims, md, **kw)[1]
            if not np.array_equal(a, b):
                changed.append(case)
        assert changed, f"{name} changes no case"
    leaf, vox, lo, dims, md = cases["pad_only"]
    assert dist_ref.field(dist_ref.keys_of_voxels(vox), leaf, lo, dims, md)[1][2, 2, 0] == 9


# (leaf, lo, dims, max_distance, accepted): each limit at its edge (pad = floor(R) + 1)
LIMIT_CASES = [(0.5, (0, 0, 0), (8192 - 2 * 3, 4, 4), 1.0, True),
               (0.5, (0, 0, 0), (8192 - 2 * 3 + 1, 4, 4), 1.0, False),
               (0.5, (0, 0, 0), (4, 8192 - 2 * 3, 4), 1.0, True),
               (0.5, (0, 0, 0), (4, 4, 8192 - 2 * 3 + 1), 1.0, False),
               (0.5, (0, 0, 0), (1, 1, 1), 512.001, False),  # ratio > 1024 (the cells limit binds first below)
               (0.25, (-(1 << 20) + 5, 0, 0), (3, 3, 3), 1.0, True),
               (0.25, (-(1 << 20) + 4, 0, 0), (3, 3, 3), 1.0, False),
               (0.25, (0, (1 << 20) - 8, 0), (3, 3, 3), 1.0, True),
               (0.25, (0, (1 << 20) - 7, 0), (3, 3, 3), 1.0, False),
               (0.2, (0, 0, 0), (512 - 6, 512 - 6, 512 - 6), 0.4, True),
               (0.2, (0, 0, 0), (512 - 6, 512 - 6, 512 - 5), 0.4, False),
               (0.2, (0, 0, 0), (4, 0, 4), 0.4, False),
               (0.2, (0, 0, 0), (4, 4, 4), 0.0, False),
               (0.2, (0, 0, 0), (4, 4, 4), float("inf"), False)]


@pytest.mark.parametrize("case", range(len(LIMIT_CASES)))
def test_limits(case):
    leaf, lo, dims, md, ok = LIMIT_CASES[case]
    assert dist_ref.box_ok(leaf, lo, dims, md) == ok


def test_pad_floor_is_caught():
    """pad = floor(R) gives the same values (see distance_reference) but accepts boxes the + 1 refuses."""
    assert any(dist_ref.box_ok(leaf, lo, dims, md, pad_floor=True) != ok for leaf, lo, dims, md, ok in LIMIT_CASES)


def small_field(leaf=0.25, md=1.0):
    keys, vox = random_target(5, n=40, span=6)
    lo, dims = (-7, -6, -8), (13, 12, 15)
    return keys, dist_ref.field(keys, leaf, lo, dims, md), lo, dims


def test_query_at_centres():
    """At cell centres (exact in fp64 at a power-of-two leaf) the query is the cell's distance, the beyond cells
    saturated at max_distance."""
    leaf, md = 0.25, 1.0
    keys, (dist, sq), lo, dims = small_field(leaf, md)
    idx = np.argwhere(np.ones(sq.shape, bool))  # z y x
    vox = idx[:, ::-1] + np.array(lo)
    d, _ = dist_ref.query(sq, leaf, lo, md, dist_ref.centres(leaf, vox))
    want = np.where(np.isinf(dist), np.float32(md), dist)[idx[:, 0], idx[:, 1], idx[:, 2]]
    assert np.array_equal(d, want)


def test_query_linear_and_gradient():
    leaf, md = 0.25, 1.0
    keys, (dist, sq), lo, dims = small_field(leaf, md)
    rng = np.random.RandomState(2)
    L = float(np.float32(leaf))
    # linear along x between two neighbouring centres
    for _ in range(50):
        v = np.array([rng.randint(0, dims[0] - 1), rng.randint(0, dims[1]), rng.randint(0, dims[2])]) + np.array(lo)
        a, b = dist_ref.centres(leaf, [v, v + [1, 0, 0]])
        t = rng.uniform(0.05, 0.95)
        p = a.astype(np.float64) + t * (b.astype(np.float64) - a.astype(np.float64))
        d, _ = dist_ref.query(sq, leaf, lo, md, np.float32(p[None]))
        da, db = dist_ref.query(sq, leaf, lo, md, np.stack([a, b]))[0]
        assert abs(float(d[0]) - (float(da) + t * (float(db) - float(da)))) <= 1e-5
    # the gradient against central differences, inside a cell (away from the kinks at cell boundaries)
    g = rng.uniform(0.2, 0.8, (300, 3)) + rng.randint(0, 1000, (300, 3)) % (np.array(dims) - 1)
    p = ((g + 0.5 + np.array(lo)) * L)
    pts = np.concatenate([p, np.zeros((300, 1))], axis=1).astype(np.float32)
    d, grad = dist_ref.query(sq, leaf, lo, md, pts)
    h = 0.01 * L
    for ax in range(3):
        e = np.zeros(4)
        e[ax] = h
        dp = dist_ref.query(sq, leaf, lo, md, (pts.astype(np.float64) + e).astype(np.float32))[0].astype(np.float64)
        dm = dist_ref.query(sq, leaf, lo, md, (pts.astype(np.float64) - e).astype(np.float32))[0].astype(np.float64)
        fd = (dp - dm) / ((pts[:, ax].astype(np.float64) + h).astype(np.float32).astype(np.float64) -
                          (pts[:, ax].astype(np.float64) - h).astype(np.float32).astype(np.float64))
        assert np.abs(fd - grad[:, ax]).max() <= 2e-3 * max(1.0, np.abs(grad[:, ax]).max())
    assert np.isfinite(grad).all() and np.abs(grad).max() > 0.5


def test_query_hull():
    """NaN just outside the hull of the cell centres; defined on it, including the last centre (i = n - 2, f = 1);
    every query NaN on a box one cell thick; NaN and infinite coordinates."""
    leaf, md = 0.25, 1.0
    keys, (dist, sq), lo, dims = small_field(leaf, md)
    L = float(np.float32(leaf))
    first = dist_ref.centres(leaf, [np.array(lo)])[0]
    last = dist_ref.centres(leaf, [np.array(lo) + np.array(dims) - 1])[0]
    pts = np.stack([first, last])
    d, _ = dist_ref.query(sq, leaf, lo, md, pts)
    assert np.isfinite(d).all()
    assert d[1] == np.where(np.isinf(dist[-1, -1, -1]), np.float32(md), dist[-1, -1, -1])
    for ax in range(3):
        for p, s in ((first, -1), (last, 1)):
            q = p.copy()
            q[ax] = np.nextafter(q[ax], np.float32(s * np.inf))
            assert np.isnan(dist_ref.query(sq, leaf, lo, md, q[None])[0]).all()
            q[ax] = p[ax] + np.float32(s * 0.5 * L)
            assert np.isnan(dist_ref.query(sq, leaf, lo, md, q[None])[0]).all()
            assert np.isfinite(dist_ref.query(sq, leaf, lo, md, q[None], hull_off_by_one=True)[0]).all() or s < 0
    bad = np.array([[np.nan, first[1], first[2], 0], [np.inf, first[1], first[2], 0], [first[0], -np.inf, 0, 0]],
                   np.float32)
    d, g = dist_ref.query(sq, leaf, lo, md, bad)
    assert np.isnan(d).all() and np.isnan(g).all()
    thin = sq[:1]  # nz = 1
    d, g = dist_ref.query(thin, leaf, lo, md, np.stack([first, first + [L, L, 0, 0]]))
    assert np.isnan(d).all() and np.isnan(g).all()


def test_query_saturates():
    """Far from every obstacle all corners are beyond: the query is max_distance and its gradient 0."""
    keys = dist_ref.keys_of_voxels([[8, 0, 0]])
    lo, dims = (10, -3, -3), (8, 7, 7)
    dist, sq = dist_ref.field(keys, 0.5, lo, dims, 2.0)
    assert (sq[:, :, 4:] == -1).all()
    p = dist_ref.centres(0.5, [[16, 0, 0], [15, 1, -1]])
    p[1, :3] += np.float32(0.1)
    d, g = dist_ref.query(sq, 0.5, lo, 2.0, p)
    assert (d == np.float32(2.0)).all() and (g == 0).all()
    # the gradient points away from the obstacle where the field is below the range
    d, g = dist_ref.query(sq, 0.5, lo, 2.0, dist_ref.centres(0.5, [[11, 0, 0]]) + np.float32([0.1, 0.05, 0.05, 0]))
    assert d[0] < 2.0 and g[0, 0] > 0


def test_query_wrong_hull_is_caught():
    leaf, md = 0.25, 1.0
    keys, (dist, sq), lo, dims = small_field(leaf, md)
    last = dist_ref.centres(leaf, [np.array(lo) + np.array(dims) - 1])[0]
    q = last + np.float32([0.5 * 0.25, 0, 0, 0])
    a = dist_ref.query(sq, leaf, lo, md, q[None])[0]
    b = dist_ref.query(sq, leaf, lo, md, q[None], hull_off_by_one=True)[0]
    assert np.isnan(a).all() and np.isfinite(b).all()


def test_voxel_box():
    from loam_velodyne_b200 import api
    lo, dims = api.voxel_box((-1.0, 0.0, 2.05), (1.0, 0.35, 2.05), 0.1)
    inv = np.float32(1.0) / np.float32(0.1)
    want_lo = np.floor(np.float32([-1.0, 0.0, 2.05]) * inv).astype(np.int32)
    want_hi = np.floor(np.float32([1.0, 0.35, 2.05]) * inv).astype(np.int32)
    assert lo.tolist() == want_lo.tolist() and dims.tolist() == (want_hi - want_lo + 1).tolist()
    assert dims[2] == 1 and lo.dtype == np.int32
    assert math.isclose(float(dims[0]), 21.0)
