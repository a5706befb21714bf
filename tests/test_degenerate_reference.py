"""CPU checks of the degeneracy handling of both Gauss-Newton loops and of the inputs the GPU tests run it on
(tests/degenerate_reference.py): the library's host 6 x 6 step on adversarial spectra against float64 and the checker,
the margins that keep the degenerate worlds degenerate, the replay and its wrong variants on the restatement, and the
restatement against the compiled reference in the tunnel."""

import numpy as np
import pytest

import degenerate_reference as dg

ODOM_ITER, MAP_ITER = 25, 10
ODOM_DELTA, MAP_DELTA = 0.1, 0.05
# |P x - x_lib| of the projected step, relative to max(1, |x_plain|): the checker's fp32 eigenvectors inverted in float64
# against the library's fp32 inverse and product (test_abi.py holds the same step to 2e-4)
PROJ_TOL = 2e-4


@pytest.fixture(scope="module")
def lidar():
    from loam_velodyne_b200 import synth
    return synth.Lidar.vlp16()


@pytest.fixture(scope="module")
def scenes():
    return {name: w[0]() for name, w in dg.WORLDS.items()}


@pytest.fixture(scope="module")
def tunnel_map():
    return dg.tunnel_map()


# ---------------------------------------------------------------------------------------------- the 6 x 6 step
@pytest.mark.parametrize("thr", [dg.ODOM_THR, dg.MAP_THR])
def test_step_on_adversarial_spectra(build_libs, checker, thr):
    """api.gn_solve on every matrix of dg.spectra(thr): the degenerate flag equals float64's lambda_min < thr outside
    the fp32 band (64 ulp of lambda_max, dg.fp32_noise_band), the plain step equals the checker's colPivHouseholderQr
    bit for bit, the projected step equals the float64 projection of the checker's eigenvectors within PROJ_TOL."""
    from loam_velodyne_b200 import api
    cases = dg.spectra(thr)
    n_flag = n_deg = n_shortcut_off = n_top = 0
    for name, A, b in cases:
        x_plain = checker.qr_solve6(A, b)
        x_later, d_later = api.gn_solve(A, b, False, thr)
        assert not d_later, name
        np.testing.assert_array_equal(x_later, x_plain, err_msg=f"{name}: plain step")
        x, deg = api.gn_solve(A, b, True, thr)
        w64 = np.linalg.eigvalsh(A.astype(np.float64))
        band = dg.fp32_noise_band(A)
        if abs(w64[0] - thr) > band:
            assert deg == bool(w64[0] < thr), (name, w64, band)
            n_flag += 1
        tr = float(np.trace(A.astype(np.float64)))
        n_shortcut_off += int(w64[0] < thr + 1e-5 * tr)  # the Cholesky shortcut cannot have answered
        n_top += int(1e-5 * tr > thr)
        P, deg_c = dg.projection(A, checker, thr)
        assert deg == deg_c, (name, w64)  # the library's eigenvalues decide as the checker's
        if not deg:
            np.testing.assert_array_equal(x, x_plain, err_msg=f"{name}: step without projection")
            continue
        n_deg += 1
        want = P @ x_plain.astype(np.float64)
        scale = max(1.0, float(np.abs(x_plain).max()))
        err = float(np.abs(x.astype(np.float64) - want).max()) / scale
        assert err <= PROJ_TOL, (name, err, x, want)
    assert n_flag >= len(cases) // 2 and n_deg >= len(cases) // 3 and n_top >= 20, (n_flag, n_deg, n_top, len(cases))
    assert n_shortcut_off >= n_deg


def test_spectra_cover_the_shortcut_edges():
    """The matrices really sit where they are meant to: per trace every listed lambda_min / thr, matrices whose
    lambda_min lies inside the shortcut's margin (thr, thr + 1e-5 tr], and sub-threshold pairs at each relative gap."""
    for thr in (dg.ODOM_THR, dg.MAP_THR):
        cases = dict((n, a) for n, a, _ in dg.spectra(thr))
        in_margin = 0
        for name, A in cases.items():
            w = np.linalg.eigvalsh(A.astype(np.float64))
            tr = float(np.trace(A.astype(np.float64)))
            in_margin += int(thr < w[0] <= thr + 1e-5 * tr)
            if name.startswith("pair:"):
                gap = float(name.split(":")[1])
                lo = w[w < thr]
                assert lo.size == 2 and abs((lo[1] - lo[0]) / lo[0] - gap) < 0.05 * gap + 1e-4 * (1 + tr / thr), (name, w)
            if name.startswith("negative"):
                assert w[0] < 0, (name, w)
            if name in ("singular", "zero_column"):
                assert abs(w[0]) <= 1e-5 * w[-1], (name, w)
        assert in_margin >= 6, in_margin


# ---------------------------------------------------------------------------------------------- the worlds
def _odom_iterator(oracle, scenes, lidar, world):
    from oracle import pydriver
    k0, start, _ = dg.ODOM_CASES[world]
    it = pydriver.OdomIterator(oracle, *dg.odom_clouds(oracle, world, scenes[world], lidar, k0))
    return it, start


@pytest.mark.parametrize("world", sorted(dg.ODOM_CASES))
def test_odometry_world_margin(oracle, scenes, lidar, world):
    """The first AtA of the odometry in each world has the recorded number of eigenvalues below 10, the largest of them
    below 10 / 4 and the smallest one above at least 4 x 10; the weakest direction is a translation."""
    it, start = _odom_iterator(oracle, scenes, lidar, world)
    r = it.iterate(0, start)
    assert r["n_selected"] >= 200
    w, V = oracle.eig_sym(r["AtA"])
    n_low, lo, hi = dg.spectrum_margin(w, dg.ODOM_THR)
    assert n_low == dg.ODOM_CASES[world][2] and lo < 0.25 and hi > 4.0, (world, w)
    assert np.abs(V[3:, 0]).max() > 0.95, (world, V[:, 0])


def test_mapping_world_margin(oracle, scenes, lidar, tunnel_map):
    """The scan-to-map loop's first AtA in the tunnel map: the recorded eigenvalues below 100 with a factor 4 margin on
    both sides; the weakest direction is the forward translation (z)."""
    from oracle import pydriver
    cq, sq = dg.map_queries(oracle, "tunnel", scenes["tunnel"], lidar, dg.MAP_SWEEP)
    assert tunnel_map[0].shape[0] > 10 and tunnel_map[1].shape[0] > 100
    r = pydriver.map_iteration(oracle, *tunnel_map, cq, sq, dg.map_start())
    assert r["n_selected"] >= 1000
    w, V = oracle.eig_sym(r["AtA"])
    n_low, lo, hi = dg.spectrum_margin(w, dg.MAP_THR)
    assert n_low == dg.MAP_N_DEGENERATE and lo < 0.25 and hi > 4.0, w
    assert abs(V[5, 0]) > 0.99, V[:, 0]


def test_sweeps_are_ragged(scenes, lidar):
    for world in dg.WORLDS:
        _, rs = dg.sweep(world, scenes[world], lidar, 0)
        assert rs.min() < rs.max() and rs.min() > 0, (world, rs)


def _replays(ne, start, drv, thr, min_sel, max_iter, delta):
    return {v: dg.replay(ne, start, drv, thr, min_sel, max_iter, delta, v) for v in dg.VARIANTS}


def _assert_variants_apart(res, what, floor):
    t, iters, deg, _ = res["carried"]
    assert deg and iters >= 3, (what, iters, deg)
    for v in dg.VARIANTS[1:]:
        d = float(np.abs(res[v][0] - t).max())
        assert d >= floor, (what, v, d)


@pytest.mark.parametrize("world", sorted(dg.ODOM_CASES))
def test_odometry_replay_variants_on_the_restatement(oracle, scenes, lidar, world):
    """The replay on the restatement's normal equations reports degenerate, takes several steps, and every wrong
    variant ends at least 1 mm / 1 mrad away from the upstream rule."""
    it, start = _odom_iterator(oracle, scenes, lidar, world)

    def ne(i, t):
        r = it.iterate(i, t)
        return r["AtA"], r["AtB"], r["n_selected"]
    _assert_variants_apart(_replays(ne, start, oracle, dg.ODOM_THR, dg.ODOM_MIN_SEL, ODOM_ITER, ODOM_DELTA),
                           world, 1e-3)


def test_mapping_replay_variants_on_the_restatement(oracle, scenes, lidar, tunnel_map):
    from oracle import pydriver
    cq, sq = dg.map_queries(oracle, "tunnel", scenes["tunnel"], lidar, dg.MAP_SWEEP)

    def ne(i, t):
        r = pydriver.map_iteration(oracle, *tunnel_map, cq, sq, t)
        return r["AtA"], r["AtB"], r["n_selected"]
    _assert_variants_apart(_replays(ne, dg.map_start(), oracle, dg.MAP_THR, dg.MAP_MIN_SEL, MAP_ITER, MAP_DELTA),
                           "map", 1e-3)


def test_replay_skips_starved_iterations(oracle):
    """Iterations below the selection floor leave the pose alone and are counted; a skipped iteration 0 means no
    degeneracy test at all."""
    A = np.diag([1.0, 2e3, 3e3, 4e3, 5e3, 6e3]).astype(np.float32)
    b = np.ones(6, np.float32)
    start = np.full(6, 0.25, np.float32)
    t, iters, deg, log = dg.replay(lambda i, t: (A, b, 9), start, oracle, 10.0, 10, 25, 0.1)
    assert iters == 25 and not deg and all(x is None for _, _, x in log)
    np.testing.assert_array_equal(t, start)
    seq = iter([9] + [10] * 24)
    t, iters, deg, log = dg.replay(lambda i, t: (A, b, next(seq)), start, oracle, 10.0, 10, 25, 0.1)
    assert not deg and log[0][2] is None and log[1][2] is not None


# ---------------------------------------------------------------------------------------------- checker vs reference
def _tunnel_pipeline(drv, scene, lidar, tunnel_map, n=4):
    p = drv.pipeline()
    p.seed_map(*tunnel_map)
    out = []
    for k in range(n):
        ok, od, aft, _ = p.sweep(*dg.sweep("tunnel", scene, lidar, k))
        out.append((ok, od.copy(), aft.copy(), p.mapping.cloud("surf_cubes").shape[0]))
    return out


def test_restatement_equals_compiled_reference_in_the_tunnel(oracle, reference, scenes, lidar, tunnel_map):
    """Whenever oracle/_ref is missing the restatement's projection is the checker: in the tunnel, where it runs, the
    restatement's pipeline equals the compiled reference's bit for bit (the bar of test_oracle.py)."""
    a = _tunnel_pipeline(oracle, scenes["tunnel"], lidar, tunnel_map)
    b = _tunnel_pipeline(reference, scenes["tunnel"], lidar, tunnel_map)
    for k, (ra, rb) in enumerate(zip(a, b)):
        assert ra[0] == rb[0] and ra[3] == rb[3], k
        np.testing.assert_array_equal(ra[1], rb[1], err_msg=f"sweep {k}: odometry")
        np.testing.assert_array_equal(ra[2], rb[2], err_msg=f"sweep {k}: mapping")
    # the forward motion is not observable: the odometry does not recover it
    assert abs(float(a[-1][1][5])) < 0.5 * dg.TUNNEL_SPEED * dg.SCAN_PERIOD * (len(a) - 1)
