"""The scan-to-scan odometry stage as the pipeline runs it, through the stage API (cloud slots -> loam_b200_odom_rebuild_last
-> loam_b200_odom_prepare -> iteration 0 of loam_b200_odom_iterate_debug, which searches): the last-sweep trees on the
cluster and the multi-launch build, both scans of the correspondence search (ring ranges and the serial fallback) and
the query hand-off, compared with a plain reference (tests/odom_reference.py, pinned to the checker by
test_odom_reference.py).  At zero twist the comparison has no slack: the closest point equal or an exact fp32 distance
tie, the second and third points equal to the reference's scans from the GPU's own closest point."""
import contextlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import odom_reference as orf

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

LIDARS = {"vlp16": 0, "hdl64": 2, "dense128": 0}  # name -> first sweep
TWIST = np.array([1.5e-3, -8e-3, 6e-4, -0.03, 0.01, -0.2], np.float32)  # one non-zero twist (rot x, y, z, pos x, y, z)
ZERO = np.zeros(6, np.float32)
CLUSTER_MAX_N = 131072  # largest cloud one 16-CTA cluster launch builds a tree over (csrc/clustersort.cuh: CS_MAX_N)


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


def _set_last(c, lc, ls):
    from loam_velodyne_b200 import api
    c.cloud_upload(api.C_ODOM_LAST_CORNER, lc)
    c.cloud_upload(api.C_ODOM_LAST_SURF, ls)
    c.odom_rebuild_last()


def _set_current(c, sharp, flat):
    from loam_velodyne_b200 import api
    c.cloud_upload(api.C_ODOM_SHARP, sharp)
    c.cloud_upload(api.C_ODOM_FLAT, flat)
    c.odom_prepare()


def _stage(c, lc, ls, sharp, flat):
    _set_last(c, lc, ls)
    _set_current(c, sharp, flat)


def _search(c, twist=ZERO):
    """Correspondence indices of one search iteration (iteration 0), sharp queries first."""
    return c.odom_iterate(twist, 0, debug=True)[3]


@pytest.fixture(scope="module")
def clouds(oracle, scene):
    from loam_velodyne_b200 import synth
    return {name: orf.last_and_current(oracle, getattr(synth.Lidar, name)(), sweep, scene, 5.0)
            for name, sweep in LIDARS.items()}


@pytest.fixture(scope="module")
def refs(clouds):
    """name -> (reference search, result at zero twist, result at TWIST)"""
    out = {}
    for name, (lc, ls, sharp, flat) in clouds.items():
        s = orf.Search(lc, ls)
        out[name] = (s, s.run(sharp, flat), s.run(sharp, flat, TWIST))
    return out


# ---------------------------------------------------------------------------------------------- real sweeps
@pytest.mark.parametrize("lidar", list(LIDARS))
def test_odom_search_per_correspondence(clouds, refs, lidar):
    from loam_velodyne_b200 import api
    lc, ls, sharp, flat = clouds[lidar]
    s, res0, res_t = refs[lidar]
    with _closing(_ctx()) as c:
        _stage(c, lc, ls, sharp, flat)
        paths = (c.debug_tree_build_path(api.TREE_ODOM_CORNER), c.debug_tree_build_path(api.TREE_ODOM_SURF))
        if lidar == "dense128":  # a last surface cloud beyond one cluster launch: the multi-launch build on its own lane
            assert ls.shape[0] > CLUSTER_MAX_N and paths[1] == api.BUILD_MULTI_LAUNCH, (ls.shape[0], paths)
        else:
            assert paths == (api.BUILD_CLUSTER_PAIR,) * 2, paths
        ind = _search(c)
        assert (ind[:, 0] >= 0).mean() > 0.8 and (ind[:, 1] >= 0).sum() > 50
        s.check(res0, ind, f"{lidar}, zero twist")
        s.check(res_t, _search(c, TWIST), f"{lidar}, twist {TWIST}", allow_near_ties=2)


def test_odom_scan_paths_agree(clouds):
    """Ring ranges (automatic) and the serial scan (forced): the same indices on every lidar and edge case, and the
    same device-resident Gauss-Newton loop (odom_solve) bit for bit, with the loop graph and without it."""
    with _closing(_ctx()) as c:
        for name, (lc, ls, sharp, flat) in list(clouds.items()) + list(orf.edge_cases().items()):
            _stage(c, lc, ls, sharp, flat)
            for twist in (ZERO, TWIST):
                got = []
                for mode in (1, 0):
                    c.debug_odom_ring_ranges(mode)
                    got.append(_search(c, twist))
                c.debug_odom_ring_ranges(1)
                np.testing.assert_array_equal(got[0], got[1], err_msg=f"{name}: ring ranges vs serial scan")
    poses = _solve_both_modes(clouds)
    for name, (auto, serial) in poses.items():
        np.testing.assert_array_equal(auto, serial, err_msg=f"{name}: odom_solve, loop graph")
        assert 1 <= auto[6] <= 25
    # the same without the loop graph (LOAM_B200_NO_LOOP_GRAPH is read once per process)
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        np.savez(os.path.join(tmp, "in.npz"), **{f"{k}_{i}": a for k, v in clouds.items() for i, a in enumerate(v)})
        env = dict(os.environ, LOAM_B200_NO_LOOP_GRAPH="1")
        env["PYTHONPATH"] = os.pathsep.join([HERE, os.path.dirname(HERE), env.get("PYTHONPATH", "")])
        r = subprocess.run([sys.executable, "-c", "import test_odom_stage as t, sys; t._solve_main(sys.argv[1])", tmp],
                           capture_output=True, text=True, timeout=600, env=env, cwd=HERE)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
        no_graph = json.load(open(os.path.join(tmp, "out.json")))
    for name, (auto, serial) in no_graph.items():
        np.testing.assert_array_equal(np.float32(auto), np.float32(serial), err_msg=f"{name}: odom_solve, no loop graph")


def _solve_both_modes(clouds):
    """name -> (pose + iterations with ring ranges, the same with the serial scan), each a 7-vector."""
    out = {}
    with _closing(_ctx()) as c:
        for name, (lc, ls, sharp, flat) in clouds.items():
            _stage(c, lc, ls, sharp, flat)
            res = []
            for mode in (1, 0):
                c.debug_odom_ring_ranges(mode)
                pose, iters = c.odom_solve(ZERO)
                res.append(np.concatenate([pose, np.float32([iters])]))
            c.debug_odom_ring_ranges(1)
            out[name] = res
    return out


def _solve_main(tmp):
    """Subprocess body of test_odom_scan_paths_agree (run with LOAM_B200_NO_LOOP_GRAPH=1)."""
    z = np.load(os.path.join(tmp, "in.npz"))
    clouds = {name: tuple(z[f"{name}_{i}"] for i in range(4)) for name in LIDARS}
    res = _solve_both_modes(clouds)
    json.dump({k: [a.tolist(), b.tolist()] for k, (a, b) in res.items()}, open(os.path.join(tmp, "out.json"), "w"))


# ---------------------------------------------------------------------------------------------- the serial fallback
@pytest.mark.parametrize("variant", ["rings_permuted", "points_moved", "rings_250_255", "rings_250_255_sorted",
                                     "ring_gaps", "negative_intensity"])
def test_odom_fallback_clouds(clouds, variant):
    """Last clouds that are not ring-ordered or carry ring ids beyond 252 (the clouds of test_odom_reference.py),
    through the stage: the serial scan (and, for ordered ones, the hand-over from the ring ranges) against the
    reference."""
    with _closing(_ctx()) as c:
        for lidar in ("vlp16", "hdl64"):
            lc, ls, sharp, flat = clouds[lidar]
            vc, vs = orf.fallback_variants(lc, ls)[variant]
            s = orf.Search(vc, vs)
            res = s.run(sharp, flat)
            _stage(c, vc, vs, sharp, flat)
            ind = _search(c)
            assert (ind[:, 0] >= 0).mean() > 0.8
            s.check(res, ind, f"{lidar}/{variant}")


# ---------------------------------------------------------------------------------------------- tree builds
def _ring_cloud(m, seed, kind="box"):
    """m points in ring order (64 rings), with queries: a 40 m box, a plane, one point repeated, or a box plus one
    outlier at 10 km."""
    rng = np.random.RandomState(seed)
    p = np.zeros((m, 4), np.float32)
    p[:, :3] = rng.uniform(-20, 20, (m, 3))
    if kind == "planar":
        p[:, 2] = np.float32(1.5)
    elif kind == "identical":
        p[:, :3] = np.float32([3.25, -1.5, 0.75])
    elif kind == "outlier":
        p[m // 2, :3] = (1.0e4, 0.0, 0.0)
    p[:, 3] = (np.arange(m) * 64 // max(m, 1)).astype(np.float32)
    return p


def _queries_near(p, n, seed):
    rng = np.random.RandomState(seed)
    if p.shape[0] == 0 or n == 0:
        return np.zeros((0, 4), np.float32)
    q = p[rng.randint(0, p.shape[0], n)].copy()
    q[:, :3] += rng.normal(0, 0.3, (n, 3)).astype(np.float32)
    q[:, 3] = np.float32(0.25)
    return q


def _knn_against_brute_force(c, slot, last, queries):
    """tree_knn on an odometry slot: distances bit-exact, every index at its own distance (indices up to ties)."""
    for k in (1, 5):
        gi, gd = c.tree_knn(slot, queries, k)
        kk = min(k, last.shape[0])
        for r in range(queries.shape[0]):
            d = orf.sq_dist(last, queries[r, :3])
            exp = np.sort(d)[:kk]
            np.testing.assert_array_equal(gd[r, :kk], exp, err_msg=f"k={k} query {r}: distances")
            assert len(set(gi[r, :kk].tolist())) == kk and (gi[r, :kk] >= 0).all()
            np.testing.assert_array_equal(d[gi[r, :kk]], gd[r, :kk], err_msg=f"k={k} query {r}: indices")
            assert (gi[r, kk:] == -1).all()


TREE_CASES = {  # name -> (corner size, surface size, kind)
    "sizes_1_7": (1, 7, "box"),
    "sizes_8_9": (8, 9, "box"),
    "sizes_5000": (5000, 6000, "box"),
    "sizes_65536_65537": (65536, 65537, "box"),
    "boundary_131072_131073": (CLUSTER_MAX_N, CLUSTER_MAX_N + 1, "box"),
    "boundary_131073_131072": (CLUSTER_MAX_N + 1, CLUSTER_MAX_N, "box"),
    "planar": (3000, 4000, "planar"),
    "identical": (2000, 2500, "identical"),
    "outlier_10km": (3000, 4000, "outlier"),
}


@pytest.mark.parametrize("case", list(TREE_CASES))
def test_odom_tree_build_paths(case):
    from loam_velodyne_b200 import api
    mc, ms, kind = TREE_CASES[case]
    lc, ls = _ring_cloud(mc, 1, kind), _ring_cloud(ms, 2, kind)
    sharp, flat = _queries_near(lc, min(mc, 200), 3), _queries_near(ls, min(ms, 200), 4)
    s = orf.Search(lc, ls)
    res = s.run(sharp, flat)
    knn_q = (_queries_near(lc, 300, 5), _queries_near(ls, 300, 6))
    results = {}
    for no_cluster in (False, True):
        with _closing(_ctx(no_cluster)) as c:
            _stage(c, lc, ls, sharp, flat)
            paths = (c.debug_tree_build_path(api.TREE_ODOM_CORNER), c.debug_tree_build_path(api.TREE_ODOM_SURF))
            if no_cluster:
                exp = (api.BUILD_MULTI_LAUNCH,) * 2
            elif max(mc, ms) <= CLUSTER_MAX_N:
                exp = (api.BUILD_CLUSTER_PAIR,) * 2
            else:  # one cloud each side of the boundary: two lanes, each tree on the path its size allows
                exp = tuple(api.BUILD_CLUSTER if m <= CLUSTER_MAX_N else api.BUILD_MULTI_LAUNCH for m in (mc, ms))
            assert paths == exp, (no_cluster, paths, exp)
            ind = _search(c)
            s.check(res, ind, f"{case}, {'multi-launch' if no_cluster else 'cluster'} build")
            results[no_cluster] = ind
            _knn_against_brute_force(c, api.TREE_ODOM_CORNER, lc, knn_q[0])
            _knn_against_brute_force(c, api.TREE_ODOM_SURF, ls, knn_q[1])
    if kind != "identical":  # (all points tie there; each build may pick another)
        np.testing.assert_array_equal(results[False], results[True], err_msg=f"{case}: cluster vs multi-launch build")


# ---------------------------------------------------------------------------------------------- hand-made edges
def test_odom_search_edges():
    cases = orf.edge_cases()
    with _closing(_ctx()) as c:
        for name, (lc, ls, sharp, flat) in cases.items():
            s = orf.Search(lc, ls)
            res = s.run(sharp, flat)
            _stage(c, lc, ls, sharp, flat)
            for mode in (1, 0):
                c.debug_odom_ring_ranges(mode)
                ind = _search(c)
                # tiny clouds: every tie of the closest point is a designed one; no slack at all
                np.testing.assert_array_equal(ind, res["ind"], err_msg=f"{name}, ring ranges {mode}")
            c.debug_odom_ring_ranges(1)


# ---------------------------------------------------------------------------------------------- hand-offs
def test_odom_query_handoff(checker, scene, clouds):
    """loam_b200_odom_adopt fills the query array; a later upload of the sharp cloud with the same count must replace
    it.  Then the transformToEnd hand-off over two sweeps: transform_to_end2, swap into the last slots, rebuild."""
    import math

    from loam_velodyne_b200 import api, synth
    lc, ls, sharp, flat = clouds["vlp16"]
    s = orf.Search(lc, ls)
    src5 = [api.C_REG_SHARP, api.C_REG_LESS_SHARP, api.C_REG_FLAT, api.C_REG_LESS_FLAT, api.C_REG_FULL]
    moved = sharp.copy()
    moved[:, :3] = np.roll(sharp[:, :3], 7, axis=0)  # other points, same count
    assert not np.array_equal(moved, sharp)
    with _closing(_ctx()) as reg, _closing(_ctx()) as c:
        for slot, pts in zip(src5, (sharp, lc, flat, ls, ls)):
            reg.cloud_upload(slot, pts)
        _set_last(c, lc, ls)
        c.odom_adopt(reg, src5)
        np.testing.assert_array_equal(c.cloud_download(api.C_ODOM_SHARP), sharp)
        c.odom_prepare()
        s.check(s.run(sharp, flat), _search(c), "adopted queries")
        c.odom_adopt(reg, src5)
        c.cloud_upload(api.C_ODOM_SHARP, moved)  # what the drop-in does after an edit of cornerPointsSharp()
        c.odom_prepare()
        s.check(s.run(moved, flat), _search(c), "sharp cloud re-uploaded after the adoption")

    # transformToEnd hand-off: the checker's odometry over three sweeps; after sweeps 1 and 2 its last clouds are
    # transformToEnd(less sharp / less flat) with its own _transform
    lidar = synth.Lidar.vlp16()
    o = checker.odom()
    sr = checker.scanreg()
    with _closing(_ctx()) as c:
        for i in range(4):
            pts, rs = synth.make_sweep(scene, lidar, i, v=(2.0, 0.0, 0.5), yaw_rate=math.radians(20.0))
            sr.process(pts, rs)
            cur = [sr.cloud(n) for n in ("sharp", "less_sharp", "flat", "less_flat", "full")]
            if i >= 2:  # the GPU searched the last clouds it made itself; the reference searches the checker's
                _set_current(c, cur[0], cur[2])
                ref_last = (o.cloud("last_corner"), o.cloud("last_surf"))
                rs_ = orf.Search(*ref_last)
                rs_.check(rs_.run(cur[0], cur[2]), _search(c), f"sweep {i}: search over the transformToEnd clouds")
            o.set_inputs(*cur)
            o.process()
            if i == 0:
                continue
            twist = o.twist("transform")
            assert np.abs(twist).max() > 1e-3
            c.cloud_upload(api.C_ODOM_LESS_SHARP, cur[1])
            c.cloud_upload(api.C_ODOM_LESS_FLAT, cur[3])
            c.cloud_transform_to_end2(api.C_ODOM_LESS_SHARP, api.C_ODOM_LESS_FLAT, twist)
            c.cloud_swap(api.C_ODOM_LESS_SHARP, api.C_ODOM_LAST_CORNER)
            c.cloud_swap(api.C_ODOM_LESS_FLAT, api.C_ODOM_LAST_SURF)
            for slot, name in ((api.C_ODOM_LAST_CORNER, "last_corner"), (api.C_ODOM_LAST_SURF, "last_surf")):
                got, ref = c.cloud_download(slot), o.cloud(name)
                assert got.shape == ref.shape
                np.testing.assert_array_equal(got[:, 3], np.trunc(got[:, 3]))  # intensity == int(intensity) exactly
                np.testing.assert_array_equal(got[:, 3], ref[:, 3])
                np.testing.assert_allclose(got[:, :3], ref[:, :3], rtol=0, atol=2e-5)  # the transformToEnd bar
            c.odom_rebuild_last()
