"""Host paths around the two Gauss-Newton iteration kernels that the stage tests do not reach: the instrumented
(map_iterate_stats) and debug (map_iterate_debug) launches of the scan-to-map kernel against the plain one on both
lookups, the device-resident loops (odom_solve, map_solve) in their chunked form without the loop graph against the
graph, bit for bit, and the number of kernel launches each of these entry points issues."""
import json
import math
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from test_map_stage import POSES, _closing, _ctx, _setup_search, stacks_src  # noqa: F401 (stacks_src: fixture)

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ZERO = np.zeros(6, np.float32)
STORE_POSE = np.asarray(POSES["yaw"], np.float32)
# (max_iter, delta_t = delta_r) per loop: the first converges before its cap, the others run into it (odometry: a
# partial last chunk and whole chunks of the chunked form)
CASES = {"odom": ((25, 2.0), (7, 0.1), (25, 0.1)), "map": ((10, 0.05), (2, 0.05))}


def _same_ne(a, b, what):
    np.testing.assert_array_equal(a["AtA"], b["AtA"], err_msg=f"{what}: AtA")
    np.testing.assert_array_equal(a["AtB"], b["AtB"], err_msg=f"{what}: AtB")
    assert (a["n_selected"], a["n_corner_selected"]) == (b["n_selected"], b["n_corner_selected"]), what


@pytest.fixture(scope="module")
def inputs(oracle, scene, map_200k, stacks_src):
    """Odometry clouds (sweeps 0 -> 1), scan-to-map queries of sweep 5 with a start pose near the truth (as
    test_gpu_parity.py), and the map + stacks of the stage-API search (as test_map_stage.py)."""
    from loam_velodyne_b200 import synth
    lidar = synth.Lidar.vlp16()
    s = oracle.scanreg()
    s.process(*synth.make_sweep(scene, lidar, 0, yaw_rate=math.radians(5.0)))
    last_c, last_s = s.cloud("less_sharp").copy(), s.cloud("less_flat").copy()
    last_c[:, 3] = np.floor(last_c[:, 3])
    last_s[:, 3] = np.floor(last_s[:, 3])
    s.process(*synth.make_sweep(scene, lidar, 1, yaw_rate=math.radians(5.0)))
    sharp, flat = s.cloud("sharp").copy(), s.cloud("flat").copy()
    s = oracle.scanreg()
    s.process(*synth.make_sweep(scene, lidar, 5, yaw_rate=math.radians(5.0)))
    cq = oracle.voxel_grid(s.cloud("less_sharp"), 0.2)
    sq = oracle.voxel_grid(s.cloud("less_flat"), 0.4)
    pos, yaw = synth.pose_at(0.6, np.array([0.0, 0.0, 1.0]), math.radians(5.0))
    start = np.asarray((0.002, yaw + 0.004, -0.003, pos[0] + 0.05, pos[1] - 0.02, pos[2] + 0.08), np.float32)
    return {"last_c": last_c, "last_s": last_s, "sharp": sharp, "flat": flat, "map_c": map_200k[0],
            "map_s": map_200k[1], "cq": cq, "sq": sq, "start": start, "stack_c": stacks_src[0], "stack_s": stacks_src[1]}


def _grid_map(c, inp):
    """Kernel-level API: the map slots' grids (GridCellLookup) and sweep 5's queries."""
    from loam_velodyne_b200 import api
    c.tree_build(api.TREE_MAP_CORNER, inp["map_c"])
    c.tree_build(api.TREE_MAP_SURF, inp["map_s"])
    c.map_set_queries(inp["cq"], inp["sq"])


def _store_map(c, inp):
    """Stage API: the persistent pools (MapCellLookup) and the down-sized stacks of one begin_sweep."""
    _setup_search(c, STORE_POSE, "fov", (inp["stack_c"], inp["stack_s"]), (inp["map_c"], inp["map_s"]))


def _counted(c, fn, *args, **kw):
    n0 = c.launch_count()
    r = fn(*args, **kw)
    return r, c.launch_count() - n0


# ---------------------------------------------------------------------------------------------- per-iteration launches
@pytest.mark.parametrize("lookup", ["grid", "store"])
def test_map_iterate_stats_and_debug(inputs, lookup):
    """The instrumented and the debug launch return the plain launch's normal equations bit for bit; each of the three
    is one kernel launch."""
    with _closing(_ctx()) as c:
        if lookup == "grid":
            _grid_map(c, inputs)
            twist = inputs["start"]
        else:
            _store_map(c, inputs)
            twist = STORE_POSE
        plain, n_plain = _counted(c, c.map_iterate, twist)
        assert plain["n_selected"] > 200
        (stats, nodes, leaves), n_stats = _counted(c, c.map_iterate_stats, twist)
        (dbg, coeff, sel), n_dbg = _counted(c, c.map_iterate, twist, debug=True)
        _same_ne(stats, plain, f"{lookup}: map_iterate_stats")
        _same_ne(dbg, plain, f"{lookup}: map_iterate_debug")
        assert nodes > 0 and leaves > 0, (nodes, leaves)
        assert (n_plain, n_stats, n_dbg) == (1, 1, 1)


def test_odom_iterate_launches(inputs):
    """The correspondence search is launched on every 5th iteration only, the iteration kernel on every one."""
    with _closing(_ctx()) as c:
        c.odom_set_last(inputs["last_c"], inputs["last_s"])
        c.odom_set_current(inputs["sharp"], inputs["flat"])
        counts = [_counted(c, c.odom_iterate, ZERO, it)[1] for it in (0, 1, 4, 5)]
        assert counts == [2, 1, 1, 2]


# ---------------------------------------------------------------------------------------------- device-resident loops
def _solves(inp):
    """name -> pose, iterations and launch-count delta of odom_solve and map_solve (grid and store lookups) in each
    of CASES."""
    out = {}

    def run(name, c, fn, twist):
        for i, (max_iter, delta) in enumerate(CASES[name.split("_")[0]]):
            (pose, iters), n = _counted(c, fn, twist, max_iter=max_iter, delta_t=delta, delta_r=delta)
            out[f"{name}_{i}"] = [float(v) for v in pose] + [int(iters), int(n)]

    with _closing(_ctx()) as c:
        c.odom_set_last(inp["last_c"], inp["last_s"])
        c.odom_set_current(inp["sharp"], inp["flat"])
        run("odom", c, c.odom_solve, ZERO)
        _grid_map(c, inp)
        run("map_grid", c, c.map_solve, inp["start"])
    with _closing(_ctx()) as c:
        _store_map(c, inp)
        run("map_store", c, c.map_solve, STORE_POSE)
    return out


def _solve_main(tmp):
    """Subprocess body of test_solve_without_loop_graph (run with LOAM_B200_NO_LOOP_GRAPH=1)."""
    z = np.load(os.path.join(tmp, "in.npz"))
    json.dump(_solves({k: z[k] for k in z.files}), open(os.path.join(tmp, "out.json"), "w"))


def _chunked_launches(name, iters, max_iter):
    """Launches of the chunked form: the init kernel, then whole chunks (5 odometry iterations with one search, 3 map
    iterations) until a header read after a chunk shows the loop done."""
    chunk = 5 if name == "odom" else 3
    n = min(max_iter, -(-iters // chunk) * chunk)
    if name == "odom":
        return 1 + sum(2 + (it % 5 == 0) for it in range(n))
    return 1 + 2 * n


def test_solve_without_loop_graph(inputs):
    graph = _solves(inputs)
    for key, r in graph.items():
        name, i = key.rsplit("_", 1)
        max_iter, iters, launches = CASES[name.split("_")[0]][int(i)][0], r[6], r[7]
        # init + gate + (search, iterate, step) or (iterate, step) per executed iteration
        assert launches == 2 + (3 if name == "odom" else 2) * iters, (key, r)
        if int(i) > 0:
            assert iters == max_iter, (key, r)
        elif name != "map_store":
            assert 1 <= iters < max_iter, (key, r)
    with tempfile.TemporaryDirectory() as tmp:
        np.savez(os.path.join(tmp, "in.npz"), **inputs)
        env = dict(os.environ, LOAM_B200_NO_LOOP_GRAPH="1")
        env["PYTHONPATH"] = os.pathsep.join([HERE, os.path.dirname(HERE), env.get("PYTHONPATH", "")])
        r = subprocess.run([sys.executable, "-c", "import test_lm_host_paths as t, sys; t._solve_main(sys.argv[1])", tmp],
                           capture_output=True, text=True, timeout=600, env=env, cwd=HERE)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
        chunked = json.load(open(os.path.join(tmp, "out.json")))
    assert chunked.keys() == graph.keys()
    for key, g in graph.items():
        ch = chunked[key]
        name = key.split("_")[0]
        np.testing.assert_array_equal(np.float32(ch[:6]), np.float32(g[:6]), err_msg=f"{key}: pose without the loop graph")
        assert ch[6] == g[6], (key, ch, g)
        assert ch[7] == _chunked_launches(name, ch[6], CASES[name][int(key.rsplit("_", 1)[1])][0]), (key, ch)
