"""CPU: the numpy restatement of the Euclidean segmentation (tests/segment_reference.py) against brute force and
scipy's kd-tree, on hand-made cases with known answers, and against deliberately wrong restatements."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

import dense_reference as dr
import segment_reference as sr


def cloud(xyz, w=1.0):
    a = np.asarray(xyz, np.float32).reshape(-1, 3)
    return np.ascontiguousarray(np.concatenate([a, np.full((a.shape[0], 1), w, np.float32)], axis=1))


def fp32_rounding_pair(tol):
    """Two points whose fp64 distance is just above tol while fp32 arithmetic puts it at or below."""
    t = np.float32(tol)
    rng = np.random.RandomState(5)
    for _ in range(100000):
        x = np.float32(rng.uniform(0.2, 0.9) * t)
        y = np.float32(np.sqrt(np.float64(t) ** 2 - np.float64(x) ** 2))
        for _ in range(4):
            d64 = np.float64(x) ** 2 + np.float64(y) ** 2
            d32 = x * x + y * y
            if d64 > np.float64(t) ** 2 and d32 <= t * t:
                return cloud([[0.0, 0.0, 0.0], [x, y, 0.0]])
            y = np.nextafter(y, np.float32(np.inf))
    raise AssertionError("no pair found")


def edge_case_clouds():
    """name -> (points, tol, min_size, max_size).  Each holds a known answer, asserted in test_hand_made_cases."""
    c = {}
    k = np.arange(60, dtype=np.float64)
    c["chain"] = (cloud(np.stack([k * 0.25, k * 0.25, k * 0.15], axis=1)), 0.5, 1, sr.INT_MAX)
    c["exact_tol"] = (cloud([[0.25, 0, 0], [0.75, 0, 0], [10.25, 0, 0],
                             [np.nextafter(np.float32(10.75), np.float32(np.inf)), 0, 0]]), 0.5, 1, sr.INT_MAX)
    c["fp32_rounding"] = (fp32_rounding_pair(1.0), 1.0, 1, sr.INT_MAX)
    lim = float(np.float32(dr.HALF) * np.float32(0.5))
    c["row_and_plane"] = (cloud([[0.1, -0.01, 0.0], [0.1, 0.01, 0.0], [3.0, 3.0, -0.01], [3.0, 3.0, 0.01],
                                 [lim - 0.3, 0.0, 0.0], [lim - 0.6, 0.0, 0.0], [-lim + 0.1, 0.25, 0.0],
                                 [-lim + 0.1, -0.2, 0.0]]), 0.5, 1, sr.INT_MAX)
    c["negative"] = (cloud([[-0.2, -0.3, -0.1], [0.1, -0.2, 0.05], [-5.1, -7.2, -3.3], [-5.3, -7.0, -3.1],
                            [-5.5, -6.8, -2.9]]), 0.5, 1, sr.INT_MAX)
    # equal sizes: A = {0, 5}, B = {1, 2}, C = {3, 4}: smallest index ranks A, B, C; largest would rank B, C, A
    c["ties"] = (cloud([[0, 0, 0], [5, 0, 0], [5.2, 0, 0], [9, 0, 0], [9.2, 0, 0], [0.2, 0, 0]]), 0.5, 1, sr.INT_MAX)
    c["filters"] = (cloud([[0, 0, 0], [3, 0, 0], [3.2, 0, 0], [6, 0, 0], [6.2, 0, 0], [6.4, 0, 0],
                           [9, 0, 0], [9.2, 0, 0], [9.4, 0, 0], [9.6, 0, 0], [9.8, 0, 0]]), 0.5, 2, 3)
    bad = [[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [3e38, 0, 0], [3e38, 0.1, 0], [-3e38, 0, 0],
           [-3e38, 0, 0.1], [lim, 0, 0], [lim + 0.1, 0, 0], [1.0, 1.0, 1.0]]
    c["non_finite_and_out_of_range"] = (cloud(bad), 0.5, 1, sr.INT_MAX)
    c["empty"] = (np.zeros((0, 4), np.float32), 0.5, 1, sr.INT_MAX)
    return c


def target_cases():
    """name -> (leaf, centroids one per voxel, tol): tol / leaf = 2.5, a pair three voxels apart within tol."""
    leaf = 0.2
    pts = cloud([[0.99 * leaf, 0.5 * leaf, 0.5 * leaf], [3.01 * leaf, 0.5 * leaf, 0.5 * leaf],
                 [10.5 * leaf, 0.5 * leaf, 0.5 * leaf], [10.5 * leaf, 3.4 * leaf, 2.1 * leaf],
                 [-4.5 * leaf, -0.5 * leaf, -3.5 * leaf]])
    return {"three_voxels": (leaf, pts, 2.5 * leaf), "four_leaves": (leaf, pts, 4.0 * leaf)}


EXPECTED = {
    "chain": [0] * 60,
    "exact_tol": [0, 0, 1, 2],
    "fp32_rounding": [0, 1],
    "row_and_plane": [0, 0, 1, 1, 2, 2, 3, 3],
    "negative": [1, 1, 0, 0, 0],
    "ties": [0, 1, 1, 2, 2, 0],
    "filters": [-1, 1, 1, 0, 0, 0, -1, -1, -1, -1, -1],
    "non_finite_and_out_of_range": [-1, -1, -1, -1, -1, -1, -1, -1, -1, 0],
    "empty": [],
}


def same_result(a, b):
    la, sa = a
    lb, sb = b
    return np.array_equal(la, lb) and all(np.array_equal(sa[f].view(np.uint8), sb[f].view(np.uint8)) for f in sa)


@pytest.mark.parametrize("name", list(edge_case_clouds()))
def test_hand_made_cases(name):
    pts, tol, mn, mx = edge_case_clouds()[name]
    labels, seg = sr.cloud_segment(pts, tol, mn, mx)
    assert labels.tolist() == EXPECTED[name]
    k = seg["size"].size
    assert k == (max(EXPECTED[name]) + 1 if EXPECTED[name] else 0)
    for s in range(k):
        members = np.nonzero(labels == s)[0]
        assert seg["size"][s] == members.size and seg["first"][s] == members.min()
        q = pts[members, :3]
        assert np.array_equal(seg["lo"][s], q.min(axis=0)) and np.array_equal(seg["hi"][s], q.max(axis=0))
        want = (q.astype(np.float64).sum(axis=0) / members.size).astype(np.float32)
        assert np.allclose(seg["centroid"][s], want, rtol=0, atol=1e-6 * (1 + np.abs(want).max()))
    assert list(seg["size"]) == sorted(seg["size"], reverse=True)


def test_target_cases():
    for name, (leaf, pts, tol) in target_cases().items():
        keys, cent = sr.target_of(pts, leaf)
        labels, seg = sr.target_segment(keys, cent, leaf, tol)
        x = cent[:, 0] / np.float32(leaf)
        pair = np.nonzero((x > 0.9) & (x < 3.1))[0]
        assert pair.size == 2 and labels[pair[0]] == labels[pair[1]] >= 0, name
        assert labels[np.argmin(cent[:, 0])] != labels[pair[0]]


def test_same_points_as_target_and_as_cloud():
    """One point per voxel at cell = tol: the target (key order) and the cloud in key order give the same bits; a
    shuffled cloud gives the same partition, sizes and bounds, with input indices."""
    rng = np.random.RandomState(11)
    tol = 0.25
    v = np.unique(rng.randint(-30, 30, (3000, 3)), axis=0)
    pts = cloud((v + rng.uniform(0.05, 0.95, v.shape)) * tol)
    keys, cent = sr.target_of(pts, tol)
    assert np.unique(keys).size == keys.size
    t = sr.target_segment(keys, cent, tol, tol)
    assert same_result(t, sr.cloud_segment(cent, tol))
    perm = rng.permutation(cent.shape[0])
    lab, seg = sr.cloud_segment(cent[perm], tol)
    pairs = np.unique(np.stack([lab, t[0][perm]], axis=1), axis=0)  # the same partition: ids in bijection
    assert pairs.shape[0] == seg["size"].size == t[1]["size"].size
    assert np.unique(pairs[:, 0]).size == np.unique(pairs[:, 1]).size == pairs.shape[0]
    for a, b in pairs:
        assert seg["size"][a] == t[1]["size"][b] and np.array_equal(seg["lo"][a], t[1]["lo"][b])
        assert seg["first"][a] == np.nonzero(lab == a)[0].min()


def clustered(n, seed, spread=4.0):
    rng = np.random.RandomState(seed)
    centres = rng.uniform(-spread, spread, (max(n // 40, 1), 3))
    p = centres[rng.randint(0, centres.shape[0], n)] + rng.normal(0, 0.3, (n, 3))
    return cloud(p)


@pytest.mark.parametrize("tol", [0.05, 0.2, 0.37])
def test_edges_equal_brute_force(tol):
    for seed in range(3):
        pts = clustered(400, seed)
        pts[::53, 1] = np.nan
        assert sr.cloud_edges(pts, tol) == sr.brute_edges(pts, tol)
    for name, (pts, t, _, _) in edge_case_clouds().items():
        assert sr.cloud_edges(pts, t) == sr.brute_edges(pts, t), name


@pytest.mark.parametrize("tol", [0.1, 0.3])
def test_edges_equal_kdtree(tol):
    pts = clustered(30000, 7, spread=20.0)
    got = sr.cloud_edges(pts, tol)
    q = pts[:, :3].astype(np.float64)
    want = cKDTree(q).query_pairs(float(np.float32(tol)))
    t2 = float(np.float32(tol)) ** 2

    def far_from_threshold(pairs):
        a = np.array(sorted(pairs), np.int64).reshape(-1, 2)
        d = q[a[:, 0]] - q[a[:, 1]]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        keep = np.abs(d2 - t2) > 1e-9 * t2
        return set(map(tuple, a[keep].tolist()))

    assert len(got) > 1000
    assert far_from_threshold(got) == far_from_threshold(want)


@pytest.mark.parametrize("variant", sr.VARIANTS)
def test_wrong_restatements_are_caught(variant):
    caught = []
    for name, (pts, tol, mn, mx) in edge_case_clouds().items():
        if not same_result(sr.cloud_segment(pts, tol, mn, mx), sr.cloud_segment(pts, tol, mn, mx, variant)):
            caught.append(name)
    for name, (leaf, pts, tol) in target_cases().items():
        keys, cent = sr.target_of(pts, leaf)
        if not same_result(sr.target_segment(keys, cent, leaf, tol),
                           sr.target_segment(keys, cent, leaf, tol, variant=variant)):
            caught.append(name)
    assert caught, variant
