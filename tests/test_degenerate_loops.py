"""Both device-resident Gauss-Newton loops where LOAM is degenerate (tests/degenerate_reference.py): the warp step on
adversarial spectra, odom_solve / map_solve in the tunnel and beside one wall against a float64 host replay (with the
wrong variants that must be told apart), the loop graph against its chunked form, the starvation gates on both sides of
their boundaries, and the pipeline with the device loops (LOAM_B200_DEVICE_LOOP=1) against the checker and the host
loop.  The tests of this file take about 10 s on an H100 80GB HBM3."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import degenerate_reference as dg

HERE = os.path.dirname(os.path.abspath(__file__))
POSE_TOL = 1e-4  # m and rad, as test_gpu_parity.py
ODOM_ITER, MAP_ITER = 25, 10
ODOM_DELTA, MAP_DELTA = 0.1, 0.05
# device pose vs the float64 replay (max over the six components), measured on an H100 80GB HBM3 at 700 W; the
# well-conditioned loops agree within 5e-6 (test_gpu_parity.py)
REPLAY_TOL = {"odom": 1e-6, "map": 1e-6}
# host loop vs device loop in the pipeline: only the sin / cos of the updated angles can differ (DESIGN.md §3); measured
# 0 on both streams on an H100 80GB HBM3 at 700 W
LOOP_FORM_TOL = 1e-6
# the tunnel stream against the checker: the forward translation is unobservable, so the step along it amplifies the
# 1e-4-relative differences of the GPU's reduction order in AtA / AtB.  Both loop forms deviate identically (measured
# up to 7.9e-4 in the odometry sums and 3.2e-3 in the mapped poses over 10 sweeps)
TUNNEL_CHECKER_TOL = 5e-3


def _ctx():
    from loam_velodyne_b200 import api
    return api.Ctx(0)


def _sub(a, idx):
    return np.ascontiguousarray(a[idx], np.float32).reshape(-1, 4)


@pytest.fixture(scope="module")
def inputs(oracle):
    """Every array the device loops run on, built once: per odometry world the last clouds and queries, the tunnel
    map, sweep MAP_SWEEP's grid queries and raw stacks, and the starved query sets (exactly 9 odometry / 49 mapping
    queries that select)."""
    from loam_velodyne_b200 import synth
    lidar = synth.Lidar.vlp16()
    out = {}
    for world, (k0, start, _) in dg.ODOM_CASES.items():
        scene = dg.WORLDS[world][0]()
        for key, a in zip(("last_c", "last_s", "sharp", "flat"), dg.odom_clouds(oracle, world, scene, lidar, k0)):
            out[f"{world}_{key}"] = a
        out[f"{world}_start"] = start
    scene = dg.tunnel()
    out["map_c"], out["map_s"] = dg.tunnel_map()
    out["cq"], out["cq_s"] = dg.map_queries(oracle, "tunnel", scene, lidar, dg.MAP_SWEEP)
    s = oracle.scanreg()
    s.process(*dg.sweep("tunnel", scene, lidar, dg.MAP_SWEEP))
    out["stack_c"], out["stack_s"] = s.cloud("less_sharp").copy(), s.cloud("less_flat").copy()
    out["map_start"] = dg.map_start()
    c = _ctx()
    try:
        c.odom_set_last(out["tunnel_last_c"], out["tunnel_last_s"])
        c.odom_set_current(out["tunnel_sharp"], out["tunnel_flat"])
        # the first 9 odometry queries that select on the whole set; on their own they select fewer (a query's
        # correspondence also depends on the other queries of its sweep), still more than none
        sel = c.odom_iterate(out["tunnel_start"], 0, debug=True)[2]
        ns = out["tunnel_sharp"].shape[0]
        pick = np.nonzero(sel == 1)[0][:dg.ODOM_MIN_SEL - 1]
        sub = (_sub(out["tunnel_sharp"], pick[pick < ns]), _sub(out["tunnel_flat"], pick[pick >= ns] - ns))
        out["starved_sharp"], out["starved_flat"] = sub
        _grid_map(c, out)
        sel = c.map_iterate(out["map_start"], debug=True)[2]
        nc = out["cq"].shape[0]
        for m in range(dg.MAP_MIN_SEL - 1, 400):
            pick = np.nonzero(sel == 1)[0][:m]
            sub = (_sub(out["cq"], pick[pick < nc]), _sub(out["cq_s"], pick[pick >= nc] - nc))
            _grid_map(c, out, *sub)
            if c.map_iterate(out["map_start"])["n_selected"] >= dg.MAP_MIN_SEL - 1:
                break
        out["starved_cq"], out["starved_sq"] = sub
    finally:
        c.close()
    return out


def _grid_map(c, inp, cq=None, sq=None):
    from loam_velodyne_b200 import api
    c.tree_build(api.TREE_MAP_CORNER, inp["map_c"])
    c.tree_build(api.TREE_MAP_SURF, inp["map_s"])
    c.map_set_queries(inp["cq"] if cq is None else cq, inp["cq_s"] if sq is None else sq)


def _store_map(c, inp):
    """The persistent pools (MapCellLookup) hold the tunnel map; begin_sweep at the start pose down-sizes the stacks."""
    import map_reference as mr
    from loam_velodyne_b200 import api
    twist = inp["map_start"]
    cen, valid, _ = mr.window(twist, (10, 5, 10))
    c.map_pool_append(0, inp["map_c"])
    c.map_pool_append(1, inp["map_s"])
    c.cloud_upload(api.C_MAP_CORNER_LAST, inp["stack_c"])
    c.cloud_upload(api.C_MAP_SURF_LAST, inp["stack_s"])
    sizes = c.map_begin_sweep(twist, cen, valid, 0.2, 0.4)
    assert sizes[0] > 10 and sizes[1] > 100, sizes


def _odom_setup(c, inp, world):
    c.odom_set_last(inp[f"{world}_last_c"], inp[f"{world}_last_s"])
    c.odom_set_current(inp[f"{world}_sharp"], inp[f"{world}_flat"])


# ---------------------------------------------------------------------------------------------- the warp step
@pytest.mark.gpu
@pytest.mark.parametrize("thr", [dg.ODOM_THR, dg.MAP_THR])
def test_warp_step_on_adversarial_spectra(ctx, thr):
    """gn_solve_warp (Ctx.debug_gn_solve) equals the host step (api.gn_solve, held against float64 and the checker in
    test_degenerate_reference.py) bit for bit on every matrix of dg.spectra, on the first and on later iterations."""
    from loam_velodyne_b200 import api
    cases = dg.spectra(thr)
    A = np.stack([a for _, a, _ in cases])
    b = np.stack([v for _, _, v in cases])
    for first in (True, False):
        xg, dgen = ctx.debug_gn_solve(A, b, first, thr)
        n_deg = 0
        for m, (name, a, v) in enumerate(cases):
            xh, dh = api.gn_solve(a, v, first, thr)
            assert bool(dgen[m]) == dh, (name, first)
            np.testing.assert_array_equal(xg[m], xh, err_msg=f"{name} first={first}")
            n_deg += int(dh)
        assert n_deg >= (len(cases) // 3 if first else 0)


# ---------------------------------------------------------------------------------------------- device loops vs replay
def _odom_replay(c, inp, world, variant="carried"):
    def ne(it, t):
        r = c.odom_iterate(t, it)
        return r["AtA"], r["AtB"], r["n_selected"]
    return dg.replay(ne, inp[f"{world}_start"], _checker(), dg.ODOM_THR, dg.ODOM_MIN_SEL, ODOM_ITER, ODOM_DELTA,
                     variant)


def _map_replay(c, inp, variant="carried"):
    def ne(it, t):
        r = c.map_iterate(t)
        return r["AtA"], r["AtB"], r["n_selected"]
    return dg.replay(ne, inp["map_start"], _checker(), dg.MAP_THR, dg.MAP_MIN_SEL, MAP_ITER, MAP_DELTA, variant)


def _checker():
    from oracle import pydriver
    return pydriver.best()


def _assert_loop_matches_replay(what, kind, dev, iters, replays):
    t, n_it, deg, _ = replays["carried"]
    dev_dist = float(np.abs(dev - t).max())
    dist = {v: float(np.abs(replays[v][0] - dev).max()) for v in dg.VARIANTS[1:]}
    print(f"\n{what}: iterations {iters}, device vs replay {dev_dist:.3g}, wrong variants " +
          ", ".join(f"{v} {d:.3g}" for v, d in dist.items()))
    assert deg, what
    assert iters == n_it and n_it >= 3, (what, iters, n_it)
    assert dev_dist <= REPLAY_TOL[kind], (what, dev, t)
    for v, d in dist.items():
        assert d >= 10 * REPLAY_TOL[kind], (what, v, d)


@pytest.mark.gpu
@pytest.mark.parametrize("world", sorted(dg.ODOM_CASES))
def test_odometry_loop_on_degenerate_input(inputs, world):
    """odom_solve carries the iteration-0 projection through every later step: same iteration count as the replay,
    pose within REPLAY_TOL, and each wrong variant at least 10 x REPLAY_TOL away."""
    c = _ctx()
    try:
        _odom_setup(c, inputs, world)
        dev, iters = c.odom_solve(inputs[f"{world}_start"], max_iter=ODOM_ITER, delta_t=ODOM_DELTA, delta_r=ODOM_DELTA)
        replays = {v: _odom_replay(c, inputs, world, v) for v in dg.VARIANTS}
    finally:
        c.close()
    _assert_loop_matches_replay(f"odom {world}", "odom", dev, iters, replays)


@pytest.mark.gpu
@pytest.mark.parametrize("lookup", ["grid", "store"])
def test_mapping_loop_on_degenerate_input(inputs, lookup):
    """map_solve in the tunnel map with the grid lookup (kernel-level API) and the store lookup (persistent pools after
    map_begin_sweep), against the replay."""
    c = _ctx()
    try:
        (_grid_map if lookup == "grid" else _store_map)(c, inputs)
        dev, iters = c.map_solve(inputs["map_start"], max_iter=MAP_ITER, delta_t=MAP_DELTA, delta_r=MAP_DELTA)
        replays = {v: _map_replay(c, inputs, v) for v in dg.VARIANTS}
    finally:
        c.close()
    _assert_loop_matches_replay(f"map {lookup}", "map", dev, iters, replays)


# ---------------------------------------------------------------------------------------------- loop forms, starvation
def _solves(inp):
    """name -> pose and iterations of every device loop of this file: the degenerate cases, and the starved ones in
    which no iteration selects enough correspondences."""
    out = {}

    def rec(name, r):
        out[name] = [float(v) for v in r[0]] + [int(r[1])]

    c = _ctx()
    try:
        for world in dg.ODOM_CASES:
            _odom_setup(c, inp, world)
            rec(f"odom_{world}", c.odom_solve(inp[f"{world}_start"], max_iter=ODOM_ITER, delta_t=ODOM_DELTA,
                                              delta_r=ODOM_DELTA))
        c.odom_set_current(inp["starved_sharp"], inp["starved_flat"])
        rec("odom_starved", c.odom_solve(inp["tunnel_start"], max_iter=ODOM_ITER))
        out["odom_starved_selected"] = int(c.odom_iterate(inp["tunnel_start"], 0)["n_selected"])
        _grid_map(c, inp)
        rec("map_grid", c.map_solve(inp["map_start"], max_iter=MAP_ITER, delta_t=MAP_DELTA, delta_r=MAP_DELTA))
        _grid_map(c, inp, inp["starved_cq"], inp["starved_sq"])
        rec("map_starved", c.map_solve(inp["map_start"], max_iter=MAP_ITER))
        out["map_starved_selected"] = int(c.map_iterate(inp["map_start"])["n_selected"])
    finally:
        c.close()
    c = _ctx()
    try:
        _store_map(c, inp)
        rec("map_store", c.map_solve(inp["map_start"], max_iter=MAP_ITER, delta_t=MAP_DELTA, delta_r=MAP_DELTA))
    finally:
        c.close()
    return out


def _solve_main(tmp):
    """Subprocess body of test_loop_forms_and_starvation (run with LOAM_B200_NO_LOOP_GRAPH=1)."""
    z = np.load(os.path.join(tmp, "in.npz"))
    json.dump(_solves({k: z[k] for k in z.files}), open(os.path.join(tmp, "out.json"), "w"))


def _subprocess(body, tmp, env_extra):
    env = dict(os.environ, **env_extra)
    env["PYTHONPATH"] = os.pathsep.join([HERE, os.path.dirname(HERE), env.get("PYTHONPATH", "")])
    r = subprocess.run([sys.executable, "-c", f"import test_degenerate_loops as t, sys; t.{body}(sys.argv[1])", tmp],
                       capture_output=True, text=True, timeout=900, env=env, cwd=HERE)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return json.load(open(os.path.join(tmp, "out.json")))


@pytest.mark.gpu
def test_loop_forms_and_starvation(inputs):
    """The chunked form (LOAM_B200_NO_LOOP_GRAPH=1) equals the loop graph bit for bit on the degenerate cases; a loop
    whose every iteration selects fewer than 10 odometry / 50 mapping correspondences (but some) returns the start pose
    bit for bit and reports max_iter iterations, in both forms."""
    graph = _solves(inputs)
    print(f"\nstarved loops select {graph['odom_starved_selected']} (odometry) and {graph['map_starved_selected']} (mapping)")
    assert 0 < graph["odom_starved_selected"] < dg.ODOM_MIN_SEL and 0 < graph["map_starved_selected"] < dg.MAP_MIN_SEL
    for key, start, cap in (("odom_starved", inputs["tunnel_start"], ODOM_ITER),
                            ("map_starved", inputs["map_start"], MAP_ITER)):
        np.testing.assert_array_equal(np.float32(graph[key][:6]), start, err_msg=key)
        assert graph[key][6] == cap, (key, graph[key])
    with tempfile.TemporaryDirectory() as tmp:
        np.savez(os.path.join(tmp, "in.npz"), **inputs)
        chunked = _subprocess("_solve_main", tmp, {"LOAM_B200_NO_LOOP_GRAPH": "1"})
    assert chunked.keys() == graph.keys()
    for key, g in graph.items():
        np.testing.assert_array_equal(np.float32(chunked[key]), np.float32(g), err_msg=f"{key}: chunked form")


# ---------------------------------------------------------------------------------------------- the starvation gates
def _odom_gate_run(odom, sweeps, n_corner, n_surf):
    """Two set_inputs / process calls; the first call's less sharp / less flat clouds (n_corner / n_surf points nearest
    the sensor) become the second call's last clouds."""
    (sh0, ls0, fl0, lf0, full0), second = sweeps
    rc = np.argsort(np.linalg.norm(ls0[:, :3], axis=1), kind="stable")[:n_corner]
    rs = np.argsort(np.linalg.norm(lf0[:, :3], axis=1), kind="stable")[:n_surf]
    odom.set_inputs(sh0, _sub(ls0, np.sort(rc)), fl0, _sub(lf0, np.sort(rs)), full0)
    odom.process()
    odom.set_inputs(*second)
    odom.process()
    return odom.twist("transform"), odom.twist("sum")


@pytest.fixture(scope="module")
def gate_sweeps(oracle):
    from loam_velodyne_b200 import synth
    lidar = synth.Lidar.vlp16()
    scene = dg.tunnel()
    out = []
    for k in (0, 1):
        s = oracle.scanreg()
        s.process(*dg.sweep("tunnel", scene, lidar, k))
        out.append(tuple(s.cloud(n).copy() for n in ("sharp", "less_sharp", "flat", "less_flat", "full")))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("n_corner,n_surf", [(10, 101), (11, 100), (11, 101)])
def test_odometry_gate(checker, gate_sweeps, n_corner, n_surf):
    """BasicLaserOdometry::process solves only with more than 10 last corner and 100 last surface points: on each side
    of either boundary the twists equal the checker's, and the loop ran (iterations > 0) exactly when both exceed it."""
    from loam_velodyne_b200 import api
    g = api.LaserOdometry()
    tg, sg = _odom_gate_run(g, gate_sweeps, n_corner, n_surf)
    tc, sc = _odom_gate_run(checker.odom(), gate_sweeps, n_corner, n_surf)
    np.testing.assert_allclose(tg, tc, rtol=0, atol=POSE_TOL)
    np.testing.assert_allclose(sg, sc, rtol=0, atol=POSE_TOL)
    opens = n_corner > 10 and n_surf > 100
    assert (g.last_iterations() > 0) == opens, g.last_iterations()
    if not opens:
        np.testing.assert_array_equal(tg, np.zeros(6, np.float32))


def _map_gate_run(m, seed, sweep):
    m.seed(*seed)
    m.set_inputs(*sweep)
    m.update_odometry(np.zeros(6, np.float32))
    m.process()
    return m.twist("aft")


@pytest.mark.gpu
@pytest.mark.parametrize("n_corner,n_surf", [(10, 101), (11, 100), (11, 101)])
def test_mapping_gate(checker, gate_sweeps, n_corner, n_surf):
    """BasicLaserMapping optimises only with more than 10 corner and 100 surface points in the cubes in view: a map
    seeded with exactly that many points nearest the sensor, on each side of either boundary."""
    from loam_velodyne_b200 import api
    mc, ms = dg.tunnel_map()
    seed = (_sub(mc, np.argsort(np.linalg.norm(mc[:, :3], axis=1), kind="stable")[:n_corner]),
            _sub(ms, np.argsort(np.linalg.norm(ms[:, :3], axis=1), kind="stable")[:n_surf]))
    sh, ls, fl, lf, full = gate_sweeps[1]
    g = api.LaserMapping()
    g.retain_from_map(True)
    ag = _map_gate_run(g, seed, (ls, lf, full))
    assert (g.cloud("corner_from_map").shape[0], g.cloud("surf_from_map").shape[0]) == (n_corner, n_surf)
    ac = _map_gate_run(checker.mapping(), seed, (ls, lf, full))
    np.testing.assert_allclose(ag, ac, rtol=0, atol=POSE_TOL)
    opens = n_corner > 10 and n_surf > 100
    assert (g.last_iterations() > 0) == opens, g.last_iterations()
    if not opens:
        np.testing.assert_array_equal(ag, np.zeros(6, np.float32))


# ---------------------------------------------------------------------------------------------- the pipeline
def _pipeline_run(streams):
    """Every stream through api.Pipeline -> {stream: (odometry sums, mapped poses, odom iterations, map iterations)}."""
    from loam_velodyne_b200 import api
    out = {}
    for name, (corner, surf, sweeps) in streams.items():
        p = api.Pipeline()
        p.seed_map(corner, surf)
        od, aft, io, im = [], [], [], []
        for pts, rs in sweeps:
            _, o, a, _ = p.sweep(pts, rs)
            od.append(o)
            aft.append(a)
            io.append(p.odom.last_iterations())
            im.append(p.mapping.last_iterations())
        out[name] = (np.array(od), np.array(aft), np.array(io), np.array(im))
    return out


def _streams(z):
    out = {}
    for name in ("vlp16", "tunnel"):
        n = int(z[f"{name}_n"])
        out[name] = (z[f"{name}_corner"], z[f"{name}_surf"], [(z[f"{name}_pts{i}"], z[f"{name}_rs{i}"]) for i in range(n)])
    return out


def _device_loop_main(tmp):
    """Subprocess body of test_pipeline_with_device_loops (run with LOAM_B200_DEVICE_LOOP=1): the sequential chain and
    run_stream on the same sweeps."""
    from loam_velodyne_b200 import api
    streams = _streams(np.load(os.path.join(tmp, "in.npz")))
    seq = _pipeline_run(streams)
    res = {name: [a.tolist() for a in r] for name, r in seq.items()}
    for name, (corner, surf, sweeps) in streams.items():
        p = api.Pipeline()
        p.seed_map(corner, surf)
        st = p.run_stream(sweeps)
        res[name + "_stream"] = [[float(v) for v in o] + [float(v) for v in a] for _, o, a in st]
    json.dump(res, open(os.path.join(tmp, "out.json"), "w"))


@pytest.mark.gpu
def test_pipeline_with_device_loops(checker, sweeps_vlp16, map_200k):
    """api.Pipeline with LOAM_B200_DEVICE_LOOP=1 (read once per process, so in a subprocess) on the VLP-16 stream and a
    tunnel stream of 10 sweeps: every pose within POSE_TOL of the checker (the tunnel's within TUNNEL_CHECKER_TOL), the same iteration counts as the host loop
    and poses within LOOP_FORM_TOL of it, and run_stream equal to the sequential chain bit for bit."""
    from loam_velodyne_b200 import synth
    lidar = synth.Lidar.vlp16()
    scene = dg.tunnel()
    streams = {"vlp16": (map_200k[0], map_200k[1], list(sweeps_vlp16)),
               "tunnel": (*dg.tunnel_map(), [dg.sweep("tunnel", scene, lidar, k) for k in range(10)])}
    arrays = {}
    for name, (corner, surf, sweeps) in streams.items():
        arrays.update({f"{name}_corner": corner, f"{name}_surf": surf, f"{name}_n": np.array(len(sweeps))})
        for i, (pts, rs) in enumerate(sweeps):
            arrays[f"{name}_pts{i}"], arrays[f"{name}_rs{i}"] = pts, rs
    host = _pipeline_run(streams)
    with tempfile.TemporaryDirectory() as tmp:
        np.savez(os.path.join(tmp, "in.npz"), **arrays)
        dev = _subprocess("_device_loop_main", tmp, {"LOAM_B200_DEVICE_LOOP": "1"})
    for name, (corner, surf, sweeps) in streams.items():
        cp = checker.pipeline()
        cp.seed_map(corner, surf)
        ref = [cp.sweep(pts, rs) for pts, rs in sweeps]
        od, aft, io, im = (np.asarray(a) for a in dev[name])
        h = host[name]
        ro, ra = np.array([r[1] for r in ref]), np.array([r[2] for r in ref])
        print(f"\n{name}: vs checker: device odom {np.abs(od - ro).max(axis=1)} map {np.abs(aft - ra).max(axis=1)}; "
              f"host odom {np.abs(h[0] - ro).max(axis=1)} map {np.abs(h[1] - ra).max(axis=1)}; "
              f"device vs host {np.abs(od - h[0]).max():.3g} {np.abs(aft - h[1]).max():.3g}; it {io.tolist()} {h[2].tolist()}")
        tol = POSE_TOL if name == "vlp16" else TUNNEL_CHECKER_TOL
        np.testing.assert_allclose(od, ro, rtol=0, atol=tol, err_msg=f"{name}: odometry")
        np.testing.assert_allclose(aft, ra, rtol=0, atol=tol, err_msg=f"{name}: mapping")
        np.testing.assert_array_equal(io, h[2], err_msg=f"{name}: odometry iterations")
        np.testing.assert_array_equal(im, h[3], err_msg=f"{name}: mapping iterations")
        d = max(float(np.abs(od - h[0]).max()), float(np.abs(aft - h[1]).max()))
        print(f"\n{name}: device loop vs host loop pose deviation {d:.3g}; iterations odom {io.tolist()} map {im.tolist()}")
        assert d <= LOOP_FORM_TOL, (name, d)
        stream = np.float32(dev[name + "_stream"])
        np.testing.assert_array_equal(stream[:, :6], np.float32(od), err_msg=f"{name}: run_stream odometry")
        np.testing.assert_array_equal(stream[:, 6:], np.float32(aft), err_msg=f"{name}: run_stream mapping")
