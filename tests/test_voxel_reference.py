"""The numpy restatements of tests/voxel_reference.py against the checker: its pcl::VoxelGrid on single clouds and the
feature stacks its mapping stage builds (to the map and back, then filtered).  The checker's VoxelGrid sorts with an
unstable std::sort, so a voxel of three or more points may be summed in another order there: centroids agree within a
few ulp, and bit for bit wherever a voxel holds at most two points.  The GPU tests (test_sort_voxel.py) then hold the
product to the restatement bit for bit.  Deliberately wrong restatements must be caught on named inputs."""
import math

import numpy as np
import pytest

import dense_reference as dr
import voxel_reference as vr

F = np.float32
LEAVES = [0.05, 0.2, 0.4, 1.0]
PLACEMENTS = {"plus": (0.7, (31.3, 1.7, 12.9)), "minus": (-2.1, (-131.3, -4.2, -57.9))}


def moved(pts, yaw, t):
    """A sweep moved into a map frame (rotation about y, translation)."""
    c, s = F(math.cos(yaw)), F(math.sin(yaw))
    p = np.array(pts, F, copy=True)
    x, z = p[:, 0].copy(), p[:, 2].copy()
    p[:, 0] = c * x + s * z + F(t[0])
    p[:, 1] = p[:, 1] + F(t[1])
    p[:, 2] = -s * x + c * z + F(t[2])
    return p


def voxel_counts(pts, leaf):
    """Points per output voxel, in output order (None when the guard trips)."""
    inv, minb, div, overflow = vr.voxel_meta(pts, leaf)
    if overflow:
        return None
    return np.unique(vr.voxel_keys(pts, inv, minb, div), return_counts=True)[1]


def assert_matches_voxel_grid(ref, pcl, pts, leaf):
    """Same voxels in the same order; centroids bit for bit where a voxel holds <= 2 points, else within as many ulp as
    the voxel has points (the error bound of a reordered float32 sum of same-sign terms, relative to the result)."""
    assert ref.shape == pcl.shape
    cnt = voxel_counts(pts, leaf)
    if cnt is None:
        assert np.array_equal(ref.view(np.uint32), pts.view(np.uint32))
        assert np.array_equal(pcl.view(np.uint32), pts.view(np.uint32))
        return
    assert cnt.shape[0] == ref.shape[0]
    sp = np.spacing(np.maximum(np.abs(ref), np.abs(pcl)).astype(F))
    ulp = np.abs(ref.astype(np.float64) - pcl.astype(np.float64)) / sp
    bad = np.flatnonzero(np.any(ulp > np.maximum(cnt, 2)[:, None], axis=1))
    assert bad.size == 0, f"{bad.size} voxels beyond their bound, first {bad[:5]}: {ulp[bad[:5]]} ulp, {cnt[bad[:5]]} points"
    small = cnt <= 2
    assert np.array_equal(ref[small].view(np.uint32), pcl[small].view(np.uint32))


@pytest.fixture(scope="module")
def sweeps(scene):
    from loam_velodyne_b200 import synth
    return {name: synth.make_sweep(scene, getattr(synth.Lidar, name)(), 3, yaw_rate=math.radians(5.0))[0]
            for name in ("vlp16", "hdl64")}


@pytest.mark.parametrize("placement", list(PLACEMENTS))
@pytest.mark.parametrize("leaf", LEAVES)
@pytest.mark.parametrize("lidar", ["vlp16", "hdl64"])
def test_voxel_grid_matches_checker(checker, sweeps, lidar, leaf, placement):
    pts = moved(sweeps[lidar], *PLACEMENTS[placement])
    ref = vr.voxel_grid(pts, leaf)
    assert_matches_voxel_grid(ref, checker.voxel_grid(pts, leaf), pts, leaf)
    if leaf == 0.05 and lidar == "vlp16":
        assert vr.voxel_meta(pts, leaf)[3], "a whole VLP-16 sweep at 5 cm trips the guard"
    else:
        assert ref.shape[0] < pts.shape[0]


@pytest.mark.parametrize("leaf", LEAVES)
def test_bit_exact_with_at_most_two_points_per_voxel(checker, sweeps, leaf):
    """Where no voxel holds three points the summation order cannot matter: equal bit for bit."""
    pts = moved(sweeps["vlp16"], *PLACEMENTS["minus"])
    pts = pts[np.all(np.abs(pts[:, :3] - pts[0, :3]) < 40.0, axis=1)]  # fits the guard at 5 cm
    inv, minb, div, overflow = vr.voxel_meta(pts, leaf)
    assert not overflow
    key = vr.voxel_keys(pts, inv, minb, div)
    order = np.argsort(key, kind="stable")
    ks = key[order]
    rank = np.arange(ks.shape[0]) - np.searchsorted(ks, ks)  # position of every point inside its voxel
    keep = np.sort(order[rank < 2])
    two = pts[keep]
    assert voxel_counts(two, leaf).max() == 2
    ref = vr.voxel_grid(two, leaf)
    assert np.array_equal(ref.view(np.uint32), checker.voxel_grid(two, leaf).view(np.uint32))


@pytest.mark.parametrize("leaf", [0.2, 0.4, 1.0])
def test_key_edges_match_checker(checker, leaf):
    pts = dr.key_edge_cloud(leaf)
    pts = pts[np.all(np.abs(pts[:, :3]) < 100.0, axis=1)]
    assert_matches_voxel_grid(vr.voxel_grid(pts, leaf), checker.voxel_grid(pts, leaf), pts, leaf)


@pytest.mark.parametrize("name", list(vr.GUARD_BOXES))
def test_guard_boxes_match_checker(checker, name):
    pts = vr.guard_box_cloud(name)
    ref = vr.voxel_grid(pts, 1.0)
    overflow = vr.voxel_meta(pts, 1.0)[3]
    assert overflow == (name == "over")
    if name == "wrap":
        # the div product passes 2^31: keys above it (the checker's int32 key overflows there, undefined in C++)
        inv, minb, div, _ = vr.voxel_meta(pts, 1.0)
        assert int(div[0]) * int(div[1]) * int(div[2]) == 2_151_680_000
        assert vr.voxel_keys(pts, inv, minb, div).max() >= 2**31
        assert ref.shape[0] < pts.shape[0]
        return
    assert_matches_voxel_grid(ref, checker.voxel_grid(pts, 1.0), pts, 1.0)


def test_order_probes_match_checker(checker):
    pts = vr.order_probe_cloud(5000, seed=3)
    assert_matches_voxel_grid(vr.voxel_grid(pts, 1.0), checker.voxel_grid(pts, 1.0), pts, 1.0)


SUM6 = (0.01, 1.3, -0.02, 3.0, 0.2, 5.0)


@pytest.mark.parametrize("sum6", [(0.0, 0.0, 0.0, 24.5, 0.0, 24.5), SUM6])
def test_stack_roundtrip_and_filter_match_checker_mapping(checker, scene, map_200k, sum6):
    """The feature stacks of the checker's mapping stage are voxel_grid(stack_roundtrip(last, tobe), leaf)."""
    from loam_velodyne_b200 import synth
    s = checker.scanreg()
    pts, rs = synth.make_sweep(scene, synth.Lidar.vlp16(), 3, yaw_rate=math.radians(5.0))
    s.process(pts, rs)
    corner, surf = s.cloud("less_sharp"), s.cloud("less_flat")
    m = checker.mapping(max_iter=0)
    m.seed(*map_200k)
    m.set_inputs(corner, surf, pts)
    m.update_odometry(np.asarray(sum6, F))
    m.process()
    tobe = m.twist("tobe")
    for last, leaf, name in ((corner, 0.2, "corner_stack_ds"), (surf, 0.4, "surf_stack_ds")):
        rt = vr.stack_roundtrip(last, tobe)
        assert not np.array_equal(rt, last)  # fp32 does not undo the round trip exactly
        assert_matches_voxel_grid(vr.voxel_grid(rt, leaf), m.cloud(name), rt, leaf)


# ---- deliberately wrong restatements


def _variant(pts, leaf, reverse=False, pairwise=False, floor64=False, guard_div=False, sort_kind="stable"):
    p = np.asarray(pts, F).reshape(-1, 4)
    inv, minb, div, overflow = vr.voxel_meta(p, leaf)
    if guard_div:
        overflow = int(div[0]) * int(div[1]) * int(div[2]) > vr.INT32_MAX
    if overflow:
        return p.copy()
    if floor64:
        ijk = [np.floor(p[:, a].astype(np.float64) / float(F(leaf))).astype(np.int64) - int(minb[a]) for a in range(3)]
        key = ((ijk[0] + ijk[1] * int(div[0]) + ijk[2] * int(div[0]) * int(div[1])) & 0xFFFFFFFF).astype(np.uint32)
    else:
        key = vr.voxel_keys(p, inv, minb, div)
    order = np.argsort(key, kind=sort_kind)
    ks, q = key[order], p[order]
    heads = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    counts = np.diff(np.r_[heads, ks.shape[0]])
    if pairwise:
        sums = np.stack([vr.pairwise_sum(q[h:h + c]) for h, c in zip(heads, counts)])
    elif reverse:
        runs = np.repeat(np.arange(heads.shape[0]), counts)
        q = q[np.lexsort((-np.arange(q.shape[0]), runs))]
        sums = vr.run_sums(q, heads, counts)
    else:
        sums = vr.run_sums(q, heads, counts)
    return sums / counts.astype(F)[:, None]


def _differs(a, b):
    return a.shape != b.shape or not np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_variant_without_mutation_is_the_restatement():
    pts = vr.order_probe_cloud(5000, seed=3)
    assert not _differs(_variant(pts, 1.0), vr.voxel_grid(pts, 1.0))


@pytest.mark.parametrize("mutation", ["reverse", "pairwise", "sort_kind"])
def test_wrong_summation_order_is_caught(mutation):
    pts = vr.order_probe_cloud(5000, seed=3)
    kw = {"sort_kind": "quicksort"} if mutation == "sort_kind" else {mutation: True}
    assert _differs(_variant(pts, 1.0, **kw), vr.voxel_grid(pts, 1.0))


def test_float64_key_is_caught():
    pts = dr.key_edge_cloud(0.2)
    pts = pts[np.all(np.abs(pts[:, :3]) < 100.0, axis=1)]
    assert _differs(_variant(pts, 0.2, floor64=True), vr.voxel_grid(pts, 0.2))


def test_guard_from_div_is_caught():
    pts = vr.guard_box_cloud("wrap")
    assert _differs(_variant(pts, 1.0, guard_div=True), vr.voxel_grid(pts, 1.0))


def test_sort_pairs_rule():
    assert [vr.sort_passes(b) for b in (1, 8, 9, 16, 24, 30, 32)] == [1, 1, 2, 2, 3, 4, 4]
    assert [vr.sort_passes(b, out_params=False) for b in (8, 16, 24, 30)] == [2, 2, 4, 4]
    rng = np.random.RandomState(1)
    k = rng.randint(0, 2**32, 5000, dtype=np.uint64).astype(np.uint32)
    v = np.arange(5000, dtype=np.int32)
    ks, vs = vr.sort_pairs(k, v, 8)
    assert np.array_equal(ks, k[vs]) and np.all(np.diff((ks & 255).astype(np.int64)) >= 0)
    lo = (ks & 255).astype(np.int64)
    assert np.all(np.diff(vs)[np.diff(lo) == 0] > 0)  # stable within equal digits
    ks16, _ = vr.sort_pairs(k, v, 8, out_params=False)  # two passes: the low 16 bits
    assert np.all(np.diff((ks16 & 0xFFFF).astype(np.int64)) >= 0) and not np.all(np.diff((ks & 0xFFFF).astype(np.int64)) >= 0)
    ks32, vs32 = vr.sort_pairs(k, v, 32)
    assert np.array_equal(ks32, np.sort(k)) and np.array_equal(vs32, np.argsort(k, kind="stable"))
