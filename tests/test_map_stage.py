"""The scan-to-map stage as the pipeline runs it, through the stage API (loam_b200_map_pool_append / _begin_sweep /
_end_sweep): the 5-NN search over the persistent cell-sorted pools (MapCellLookup, csrc/mapstore.cuh), with and
without cell pruning, and the per-sweep map update, each compared with a plain reference (tests/map_reference.py,
pinned to the checker by test_map_reference.py) from the same state and pose, so no slack is needed."""
import contextlib
import math
import os

import numpy as np
import pytest

import map_reference as mr

pytestmark = pytest.mark.gpu

LEAVES = (0.2, 0.4)
R = np.float32(1.0 - 1.0 / math.sqrt(2.0))  # two axes at this distance from a cell corner: d^2 = 1 within an ulp

POSES = {  # (rot_x, rot_y, rot_z, x, y, z); zero rotations keep crafted queries exact through the stack round trip
    "cube_corner": (0.0, 0.0, 0.0, 24.5, 0.0, 24.5),
    "x_minus_75": (0.0, 0.0, 0.0, -74.5, 0.0, -20.5),
    "yaw": (0.01, 1.3, -0.02, 3.0, 0.2, 5.0),
}
WINDOWS = ["fov", "all125", "checkerboard", "rolled"]


def _ctx(no_cluster=False):
    from loam_velodyne_b200 import api
    old = os.environ.get("LOAM_B200_NO_CLUSTER")
    if no_cluster:
        os.environ["LOAM_B200_NO_CLUSTER"] = "1"
    try:
        return api.Ctx(0)
    finally:
        if no_cluster:
            if old is None:
                del os.environ["LOAM_B200_NO_CLUSTER"]
            else:
                os.environ["LOAM_B200_NO_CLUSTER"] = old


@contextlib.contextmanager
def _closing(c):
    try:
        yield c
    finally:
        c.close()


def _face_lattice(twist):
    """Map points on integer coordinates around the sensor (cube faces x = 25 / -75 and z = 25 among them)."""
    bx, bz = math.floor(twist[3]), math.floor(twist[5])
    g = np.mgrid[bx - 4:bx + 5, -1:3, bz - 4:bz + 5].reshape(3, -1).T.astype(np.float32)
    return np.concatenate([g, np.full((g.shape[0], 1), 7.0, np.float32)], axis=1)


def _face_queries(twist):
    """Sensor-frame stack points whose map-frame position lies exactly on a cell face, 1 ulp below one, or at
    1 - 1/sqrt(2) (+- 2 ulp) from two faces, so that the cell-corner point of a diagonal neighbour is at d^2 = 1 +- ulp.
    Exact only for poses without rotation (the stack round trip is then exact)."""
    pos = np.asarray(twist[3:], np.float32)
    fr = []
    for k in range(-2, 3):
        fr.append(np.float32(R + np.float32(k) * np.spacing(R)))
    out = []
    cx0, cz0 = math.floor(pos[0]), math.floor(pos[2])
    i = 0
    for dx in (-3, -1, 1, 3):
        for dz in (-3, -1, 1, 3):
            for y, fy in ((0.0, np.float32(0.5)), (1.0, R)):
                x = np.float32(cx0 + dx)
                z = np.float32(cz0 + dz)
                mode = i % 4
                if mode == 0:
                    mx, mz = x, z + fr[i % 5]
                elif mode == 1:
                    mx, mz = np.nextafter(x, np.float32(-np.inf)), z + np.float32(0.5)
                else:
                    mx, mz = x + fr[i % 5], z + fr[(i + 2) % 5]
                out.append((np.float32(mx), np.float32(y) + fy, np.float32(mz)))
                i += 1
    m = np.asarray(out, np.float32)
    s = np.zeros((m.shape[0], 4), np.float32)
    s[:, :3] = m - pos  # exact (see docstring)
    s[:, 3] = 3.0
    return s


def _window(kind, twist, cen0):
    cen, valid, _ = mr.window(twist, cen0)
    if kind in ("fov", "rolled"):
        return cen, valid
    p = np.asarray(twist[3:], np.float64)
    centre = [int((p[a] + 25.0) / 50.0) + cen[a] - (1 if p[a] + 25.0 < 0 else 0) for a in range(3)]
    cubes = []
    for i in range(centre[0] - 2, centre[0] + 3):
        for j in range(centre[1] - 2, centre[1] + 3):
            for k in range(centre[2] - 2, centre[2] + 3):
                if kind == "checkerboard" and (i + j + k) % 2:
                    continue
                if 0 <= i < mr.W and 0 <= j < mr.H and 0 <= k < mr.D:
                    cubes.append(i + mr.W * j + mr.W * mr.H * k)
    return cen, cubes


@pytest.fixture(scope="module")
def stacks_src(oracle, scene):
    from loam_velodyne_b200 import synth
    s = oracle.scanreg()
    pts, rs = synth.make_sweep(scene, synth.Lidar.vlp16(), 3, yaw_rate=math.radians(5.0))
    s.process(pts, rs)
    return s.cloud("less_sharp"), s.cloud("less_flat")


def _ties(checker, from_map, q_map):
    """Queries whose 6 nearest map points (within 1 m) contain two at exactly the same distance."""
    if from_map.shape[0] < 6:
        return np.zeros(q_map.shape[0], bool)
    _, d2 = checker.knn(from_map, q_map, 6)
    eq = (d2[:, 1:] == d2[:, :-1]) & (d2[:, :-1] < 1.0)
    return eq.any(axis=1)


def _reach_clusters(twist, n=24):
    """Isolated 5-point clusters in free space (y = 40 m) whose fifth neighbour sits at the corner of the diagonal cell
    (+1, +1, 0), at squared distance 0.991 .. 0.999 from the query: only a search that probes that cell finds five
    neighbours within 1 m and selects the query (line clusters for corner queries, plane clusters for surface ones).
    Returns (corner map, surface map, corner queries, surface queries), queries in the sensor frame."""
    pos = np.asarray(twist[3:], np.float32)
    out = [[], [], [], []]
    for i in range(n):
        r2 = 0.991 + 0.008 * i / (n - 1)
        f = 1.0 - math.sqrt(r2 / 2.0)
        for kind, z in ((0, 22.5), (1, 26.5)):
            X = math.floor(pos[0]) - n + 2 * i
            q = np.array([X + f, 40.0 + f, z], np.float32)
            far = np.array([X + 1.0, 41.0, z], np.float32)
            if kind == 0:
                d = (far - q) / np.linalg.norm(far - q)
                near = [q + np.float32(t) * d for t in (-0.25, -0.12, 0.12, 0.3)]
            else:
                near = [q + np.array(o, np.float32) for o in ((-0.2, 0, 0), (0, -0.2, 0), (-0.3, -0.25, 0), (0.1, -0.1, 0))]
            for p in near + [far]:
                out[kind].append((*p.astype(np.float32), 5.0))
            out[2 + kind].append((*(q - pos), 77.0))  # marks the query in the down-sized stack
    return [np.asarray(o, np.float32) for o in out]


def _setup_search(c, twist, win_kind, stacks_src, map_pts, extra_queries=True, clusters=False):
    """Seed both pools, upload the stacks, begin a sweep; returns everything a search test compares."""
    from loam_velodyne_b200 import api
    corner, surf = map_pts
    lat = _face_lattice(twist)
    seed = (np.concatenate([corner, lat]), np.concatenate([surf, lat]))
    if clusters:
        cm, sm, cq, sq = _reach_clusters(twist)
        seed = (np.concatenate([seed[0], cm]), np.concatenate([seed[1], sm]))
        stacks_src = (np.concatenate([stacks_src[0], cq]), np.concatenate([stacks_src[1], sq]))
    cen0 = (13, 4, 6) if win_kind == "rolled" else (10, 5, 10)
    cen, valid = _window(win_kind, twist, cen0)
    maps = (mr.CubeMap(cen0), mr.CubeMap(cen0))
    for kind in (0, 1):
        c.map_pool_append(kind, seed[kind])
        maps[kind].add(seed[kind])
        maps[kind].roll_to(cen)
    fq = _face_queries(twist) if extra_queries else np.zeros((0, 4), np.float32)
    c.cloud_upload(api.C_MAP_CORNER_LAST, np.concatenate([stacks_src[0], fq]))
    c.cloud_upload(api.C_MAP_SURF_LAST, np.concatenate([stacks_src[1], fq]))
    c.map_debug_from_map(True)
    sizes = c.map_begin_sweep(twist, cen, valid, *LEAVES)
    fm = [maps[k].from_map(valid) for k in (0, 1)]
    stacks = (c.cloud_download(api.C_MAP_CORNER_STACK_DS), c.cloud_download(api.C_MAP_SURF_STACK_DS))
    return sizes, fm, stacks, valid


def _assert_same_search(a, b, what):
    np.testing.assert_array_equal(a[2], b[2], err_msg=f"{what}: selection")
    np.testing.assert_array_equal(a[1], b[1], err_msg=f"{what}: coefficients")
    np.testing.assert_array_equal(a[0]["AtA"], b[0]["AtA"], err_msg=f"{what}: AtA")
    np.testing.assert_array_equal(a[0]["AtB"], b[0]["AtB"], err_msg=f"{what}: AtB")


@pytest.mark.parametrize("pose_name", list(POSES))
@pytest.mark.parametrize("win_kind", WINDOWS)
def test_store_search_per_correspondence(oracle, checker, stacks_src, map_200k, win_kind, pose_name):
    """MapCellLookup (the pipeline's search) against the reference iteration and against GridCellLookup."""
    from loam_velodyne_b200 import api
    from oracle import pydriver
    twist = np.asarray(POSES[pose_name], np.float32)
    with _closing(_ctx()) as c:
        sizes, fm, stacks, valid = _setup_search(c, twist, win_kind, stacks_src, map_200k)
        assert sizes[0] == fm[0].shape[0] and sizes[1] == fm[1].shape[0]  # the <= 10 / <= 100 gate reads these
        assert sizes[2] == stacks[0].shape[0] and sizes[3] == stacks[1].shape[0]
        for k, slot in ((0, api.C_MAP_CORNER_FROM_MAP), (1, api.C_MAP_SURF_FROM_MAP)):
            np.testing.assert_array_equal(mr.sorted_rows(c.cloud_download(slot)), mr.sorted_rows(fm[k]))
        store = c.map_iterate(twist, debug=True)
        ref = pydriver.map_iteration(oracle, fm[0], fm[1], stacks[0], stacks[1], twist)
        assert ref["n_selected"] > 200
        ne, coeff, sel = store
        mism = int((sel != ref["selected"]).sum())
        assert mism <= 2, f"{mism} selection mismatches against the reference"
        both = (sel == 1) & (ref["selected"] == 1)
        np.testing.assert_allclose(coeff[both], ref["coeff"][both], rtol=0, atol=2e-6)
        rel = lambda a, b: np.abs(a - b).max() / max(np.abs(b).max(), 1e-12)
        assert rel(ne["AtA"], ref["AtA"]) <= 1e-4 and rel(ne["AtB"], ref["AtB"]) <= 1e-4
        # the same queries over the bounding-box grid of the kernel-level path
        c.tree_build(api.TREE_MAP_CORNER, fm[0])
        c.tree_build(api.TREE_MAP_SURF, fm[1])
        c.map_set_queries(stacks[0], stacks[1])
        grid = c.map_iterate(twist, debug=True)
        differ = (grid[2] != sel) | np.any(grid[1] != coeff, axis=1)
        if differ.any():
            pose = mr.Pose(twist)
            nc = stacks[0].shape[0]
            tie = np.concatenate([_ties(checker, fm[0], pose.to_map(stacks[0])),
                                  _ties(checker, fm[1], pose.to_map(stacks[1]))])
            assert tie[differ].all(), f"queries {np.flatnonzero(differ & ~tie)[:10]} differ without a distance tie (nc={nc})"
            assert rel(grid[0]["AtA"], ne["AtA"]) <= 1e-5
        else:
            _assert_same_search(store, grid, "store vs grid")


def _prune_pair(c, twist):
    c.debug_map_prune(0)
    off = c.map_iterate(twist, debug=True)
    c.debug_map_prune(1)
    on = c.map_iterate(twist, debug=True)
    c.debug_map_prune(-1)
    auto = c.map_iterate(twist, debug=True)
    return off, on, auto


def test_store_search_pruning_is_exact(stacks_src, map_200k):
    twist = np.asarray(POSES["cube_corner"], np.float32)
    with _closing(_ctx()) as c:
        _, fm, stacks, _ = _setup_search(c, twist, "all125", stacks_src, map_200k, clusters=True)
        off, on, auto = _prune_pair(c, twist)
        assert off[0]["n_selected"] > 200
        # every cluster query found its fifth neighbour in the diagonal cell and was selected
        mark = np.concatenate([stacks[0][:, 3], stacks[1][:, 3]]) == 77.0
        assert mark.sum() == 48 and off[2][mark].all(), off[2][mark]
        _assert_same_search(off, on, "pruning off vs on (200 k map)")
        _assert_same_search(off, auto, "pruning off vs auto (200 k map)")


def test_store_search_above_l2_threshold(oracle, stacks_src, scene):
    """A map beyond half of L2: the automatic mode prunes; same result as without pruning and as the reference."""
    import torch
    from loam_velodyne_b200 import synth
    from oracle import pydriver
    l2 = torch.cuda.get_device_properties(0).L2_cache_size
    n = int(l2 // 2 // 16 * 1.15)
    corner, surf = synth.make_map(scene, n)
    assert corner.shape[0] + surf.shape[0] > l2 // 2 // 16  # prune's automatic threshold
    twist = np.asarray(POSES["cube_corner"], np.float32)
    with _closing(_ctx()) as c:
        sizes, fm, stacks, _ = _setup_search(c, twist, "all125", stacks_src, (corner, surf), clusters=True)
        off, on, auto = _prune_pair(c, twist)
        _assert_same_search(off, on, "pruning off vs on (map above L2 / 2)")
        _assert_same_search(off, auto, "pruning off vs auto (map above L2 / 2)")
        ref = pydriver.map_iteration(oracle, fm[0], fm[1], stacks[0], stacks[1], twist)
        assert ref["n_selected"] > 200
        assert int((auto[2] != ref["selected"]).sum()) <= 2
        both = (auto[2] == 1) & (ref["selected"] == 1)
        np.testing.assert_allclose(auto[1][both], ref["coeff"][both], rtol=0, atol=2e-6)


# ---------------------------------------------------------------------------------------------- map update in lock step
def _voxel_keys(p, leaf):
    inv = np.float32(1.0) / np.float32(leaf)
    return np.floor(p[:, :3] * inv).astype(np.int64)


def _compare_maps(pool, ref: mr.CubeMap, valid, leaf, what):
    """Same cubes, same number of points per cube; valid cubes: the same voxels, centroids within 4 ulp of the largest
    coordinate; every other cube bit-identical."""
    got = mr.CubeMap(ref.cen)
    got.add(pool)
    assert got.indices() == ref.indices(), f"{what}: cube sets differ"
    vset = set(int(v) for v in valid)
    for idx in ref.indices():
        g, r = got.cube(idx), ref.cube(idx)
        assert g.shape == r.shape, f"{what}: cube {idx}: {g.shape[0]} points, reference {r.shape[0]}"
        if idx not in vset:
            np.testing.assert_array_equal(mr.sorted_rows(g), mr.sorted_rows(r), err_msg=f"{what}: cube {idx}")
            continue
        kg, kr = _voxel_keys(g, leaf), _voxel_keys(r, leaf)
        # by voxel, then by position (a voxel may hold two points: a centroid that rounded into it, see
        # test_map_update_edges)
        og = np.lexsort(np.concatenate([g[:, :3].T[::-1], kg.T[::-1]]))
        orr = np.lexsort(np.concatenate([r[:, :3].T[::-1], kr.T[::-1]]))
        np.testing.assert_array_equal(kg[og], kr[orr], err_msg=f"{what}: cube {idx}: voxel sets")
        gg, rr = g[og], r[orr]
        tol = 4 * np.spacing(np.abs(rr).max(axis=1))
        bad = np.abs(gg - rr).max(axis=1) > tol
        assert not bad.any(), f"{what}: cube {idx}: {bad.sum()} centroids off, e.g. {gg[bad][:2]} vs {rr[bad][:2]}"


def _lockstep_plan(map_200k):
    """Steps (predicted twist, optimised twist, corner stack input, surface stack input, points appended before)."""
    corner, surf = map_200k
    rng = np.random.RandomState(11)
    far = np.zeros((4000, 4), np.float32)
    far[:, 0] = rng.uniform(-560, 560, 4000)
    far[:, 1] = rng.uniform(-300, 300, 4000)
    far[:, 2] = rng.uniform(-560, 560, 4000)
    late = np.zeros((3000, 4), np.float32)  # raw points in a cube that first comes into view at step 4
    late[:, 0] = rng.uniform(60, 120, 3000)
    late[:, 1] = rng.uniform(-2, 3, 3000)
    late[:, 2] = rng.uniform(-20, 20, 3000)
    empty = np.zeros((0, 4), np.float32)
    d = np.array([0.003, -0.01, 0.002, 0.05, -0.02, 0.04], np.float32)
    poses = [
        (0.0, 0.2, 0.0, 0.5, 0.0, 0.5),
        (0.01, 1.3, -0.02, 3.0, 0.2, 5.0),
        (0.0, 2.4, 0.0, 24.5, 0.0, 24.5),
        (0.0, -1.1, 0.0, -74.5, 0.3, -20.5),
        (0.0, 0.0, 0.0, 70.0, 0.0, 0.0),
        (0.02, 3.0, 0.0, -380.0, 0.0, 0.0),   # grid rolls by +1: inserts land in far / new cubes
        (0.0, -2.9, 0.0, 380.0, 0.0, 0.0),    # rolls by -2
        (0.0, 0.3, 0.0, 1.0, 0.0, -2.0),
        (0.0, 0.1, 0.0, 2.0, 0.0, -1.0),
    ]
    steps = []
    for i, p in enumerate(poses):
        pred = np.asarray(p, np.float32)
        steps.append(dict(pred=pred, opt=pred + d * np.float32(1 + i % 3),
                          append=(far[:2000], far[2000:]) if i == 0 else ((empty, late) if i == 3 else None),
                          empty=(i == 7)))
    return (corner, surf), steps


@pytest.mark.parametrize("no_cluster", [False, True], ids=["cluster", "no_cluster"])
@pytest.mark.parametrize("asynchronous", [False, True], ids=["sync", "async"])
def test_map_update_lockstep(checker, stacks_src, map_200k, asynchronous, no_cluster):
    from loam_velodyne_b200 import api
    seed, steps = _lockstep_plan(map_200k)
    cen = (10, 5, 10)
    launches = []
    with _closing(_ctx(no_cluster)) as c:
        for kind in (0, 1):
            c.map_pool_append(kind, seed[kind])
        filtered_max = 0
        rolls = set()
        for n, st in enumerate(steps):
            if st["append"] is not None:
                for kind in (0, 1):
                    if st["append"][kind].shape[0]:
                        c.map_pool_append(kind, st["append"][kind])
            # the reference starts from the GPU's own pools
            maps = (mr.CubeMap(cen), mr.CubeMap(cen))
            for kind, slot in ((0, api.C_MAP_CORNER_POOL), (1, api.C_MAP_SURF_POOL)):
                maps[kind].add(c.cloud_download(slot))
            new_cen, valid, _ = mr.window(st["pred"], cen)
            rolls.add(tuple(int(a - b) for a, b in zip(new_cen, cen)))
            src = (np.zeros((0, 4), np.float32),) * 2 if st["empty"] else stacks_src
            c.cloud_upload(api.C_MAP_CORNER_LAST, src[0])
            c.cloud_upload(api.C_MAP_SURF_LAST, src[1])
            l0 = c.launch_count()
            sizes = c.map_begin_sweep(st["pred"], new_cen, valid, *LEAVES)
            stacks = (c.cloud_download(api.C_MAP_CORNER_STACK_DS), c.cloud_download(api.C_MAP_SURF_STACK_DS))
            _, fm = mr.sweep_update(maps, LEAVES, st["pred"], st["opt"], stacks, checker.voxel_grid)
            assert sizes[0] == fm[0].shape[0] and sizes[1] == fm[1].shape[0], f"step {n}: from-map sizes"
            filtered_max = max(filtered_max, int(sizes[1]) + int(sizes[3]))
            c.map_end_sweep(st["opt"], asynchronous=asynchronous)
            pools = (c.cloud_download(api.C_MAP_CORNER_POOL), c.cloud_download(api.C_MAP_SURF_POOL))
            launches.append(c.launch_count() - l0)
            for kind in (0, 1):
                _compare_maps(pools[kind], maps[kind], valid, LEAVES[kind], f"step {n} kind {kind}")
            cen = new_cen
    assert filtered_max > 131072, "the first in-view sweep should sort more than 131 072 points (onesweep sort)"
    assert (1, 0, 0) in rolls and (-2, 0, 0) in rolls
    if no_cluster:
        with _closing(_ctx()) as ref:  # the multi-launch path really ran: more launches for the same first step
            for kind in (0, 1):
                ref.map_pool_append(kind, seed[kind])
                ref.map_pool_append(kind, steps[0]["append"][kind])
            cen0, valid0, _ = mr.window(steps[0]["pred"], (10, 5, 10))
            ref.cloud_upload(api.C_MAP_CORNER_LAST, stacks_src[0])
            ref.cloud_upload(api.C_MAP_SURF_LAST, stacks_src[1])
            l0 = ref.launch_count()
            ref.map_begin_sweep(steps[0]["pred"], cen0, valid0, *LEAVES)
            ref.map_end_sweep(steps[0]["opt"], asynchronous=asynchronous)
            ref.cloud_download(api.C_MAP_SURF_POOL)
            assert launches[0] > ref.launch_count() - l0, (launches[0], ref.launch_count() - l0)


# ---------------------------------------------------------------------------------------------- hand-made update edges
def test_map_update_edges(checker):
    """A 0.4 m voxel straddling a 1 m cell face whose filtered point sits in the neighbouring cell; points exactly on
    cube faces (x = 25, -25, -75 and the store_cell quirk at -75) and on cell faces; inserts next to them."""
    from loam_velodyne_b200 import api
    f32 = np.float32
    twist = np.zeros(6, np.float32)
    seed = []
    for x in (25.0, -25.0, -75.0, 1.1, 3.0, -3.0):
        for y in (-1.0, 0.0):
            for z in (0.0, 25.0, -25.0, 2.2):
                seed.append((x, y, z, 1.0))
    seed = np.asarray(seed, f32)
    # n raw points whose fp32 centroid rounds up into the next voxel, found by brute force next to x = -53.2, plus one
    # point of that next voxel: the first filter leaves two points in one voxel, the reference's next filter of the cube
    # merges them although no new point arrives there
    crossing = []
    for leaf in LEAVES:
        inv = f32(1.0) / f32(leaf)
        face = mr.voxel_face(int(np.floor(f32(-53.2) * inv)), leaf)
        v, n = mr.first_crossing(face, -1, lambda x: np.floor(x * inv).astype(np.int64), n_max=8)
        pts = [(v, 0.1, 0.1, 4.0)] * n + [(face + f32(0.5) * f32(leaf), 0.1, 0.1, 6.0)]
        crossing.append((np.asarray(pts, f32), face, leaf))
    # stack points (sensor frame = map frame, identity pose): into the voxels of the seeded points from the other
    # side of a cell face, on the faces themselves, and just below them
    ins = []
    for x in (0.9, 24.9, -25.1, -75.1, 2.9, -3.1, 25.0, -25.0, -75.0,
              float(np.nextafter(f32(25.0), f32(-np.inf))), float(np.nextafter(f32(-75.0), f32(-np.inf)))):
        for y in (-1.0, 0.0):
            for z in (0.0, 25.0, -25.0, 2.2):
                ins.append((x, y + 0.05, z + 0.05, 2.0))
    ins = np.asarray(ins, f32)
    cen = (10, 5, 10)
    with _closing(_ctx()) as c:
        for kind in (0, 1):
            c.map_pool_append(kind, np.concatenate([seed, crossing[kind][0]]))
        empty = np.zeros((0, 4), f32)
        for step, (stack, opt) in enumerate(((empty, twist), (ins, twist), (ins[::-1].copy(), twist), (empty, twist))):
            maps = (mr.CubeMap(cen), mr.CubeMap(cen))
            for kind, slot in ((0, api.C_MAP_CORNER_POOL), (1, api.C_MAP_SURF_POOL)):
                maps[kind].add(c.cloud_download(slot))
            _, valid = _window("all125", twist, cen)
            c.cloud_upload(api.C_MAP_CORNER_LAST, stack)
            c.cloud_upload(api.C_MAP_SURF_LAST, stack)
            c.map_begin_sweep(twist, cen, valid, *LEAVES)
            stacks = (c.cloud_download(api.C_MAP_CORNER_STACK_DS), c.cloud_download(api.C_MAP_SURF_STACK_DS))
            mr.sweep_update(maps, LEAVES, twist, opt, stacks, checker.voxel_grid)
            c.map_end_sweep(opt)
            for kind, slot in ((0, api.C_MAP_CORNER_POOL), (1, api.C_MAP_SURF_POOL)):
                pool = c.cloud_download(slot)
                _compare_maps(pool, maps[kind], valid, LEAVES[kind], f"step {step} kind {kind}")
                _, face, leaf = crossing[kind]
                near = (pool[:, 0] >= face - leaf) & (pool[:, 0] < face + leaf) & (np.abs(pool[:, 1] - 0.1) < 0.01)
                landed = pool[near & (np.floor(pool[:, 0] * (f32(1.0) / f32(leaf))) == np.floor(face * (f32(1.0) / f32(leaf))))]
                assert near.sum() == landed.shape[0] == (2 if step == 0 else 1), (step, kind, pool[near])
                if step == 1 and kind == 1:
                    # the straddling voxel [0.8, 1.2) of x: one point, the centroid of the old and the new one
                    sel = (pool[:, 0] > 0.7) & (pool[:, 0] < 1.3) & (np.abs(pool[:, 1] + 1.0) < 0.2) & (np.abs(pool[:, 2]) < 0.2)
                    assert sel.sum() == 1, pool[sel]
