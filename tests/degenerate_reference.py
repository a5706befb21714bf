"""Inputs on which LOAM's degeneracy handling runs, and the float64 loop replay the device-resident Gauss-Newton loops
are held against (csrc/lmstep.cuh: gn_solve; csrc/lmstep_warp.cuh: gn_solve_warp; BasicLaserOdometry.cpp:559-622,
BasicLaserMapping.cpp:867-922).

The rule both loops follow: on iteration 0 only, take the eigenvalues of AtA (ascending); zero the ROWS of the
eigenvector matrix copy V2 that belong to the leading eigenvalues below thr (10 odometry, 100 mapping); P = V^-1 V2;
while the sweep is degenerate every step x of the plain solve is replaced by P x, iteration 0 included.  An iteration
that selects fewer than 10 (odometry) / 50 (mapping) correspondences is skipped and leaves the pose unchanged; when
iteration 0 is skipped the degeneracy test never runs.

  * tunnel(): two solid walls, floor and ceiling along z; only the forward translation is unobservable;
  * wall_and_ground(): one wall at z = 3.5 beside a sensor moving along x, and the ground; only the x translation is
    unobservable;
  * tunnel_map(): surface lattice on the tunnel's walls, floor and ceiling and corner points along its four creases;
  * spectra(): 6 x 6 AtA with chosen eigenvalues around the threshold, rounded to fp32;
  * replay(): the loop with oracle-side solves and a float64 projection, plus the deliberately wrong variants.
Which directions are degenerate is not assumed anywhere: the tests assert it from the eigen-decomposition.
"""
import math

import numpy as np

from loam_velodyne_b200 import synth

F = np.float32
TUNNEL_HALF_WIDTH = 3.5
TUNNEL_TOP = 4.0
TUNNEL_SPEED = 1.5  # m/s along the unobservable axis
SCAN_PERIOD = 0.1
MAX_RANGE = 60.0
ODOM_THR, MAP_THR = 10.0, 100.0
ODOM_MIN_SEL, MAP_MIN_SEL = 10, 50


def tunnel():
    """Walls x in [-30, -3.5] and [3.5, 30] for |z| <= 400, floor y = -1.8, ceiling y = 4 (the enclosing room's top)."""
    h = TUNNEL_HALF_WIDTH
    boxes = np.array([[-30.0, -h, -synth.SENSOR_HEIGHT, TUNNEL_TOP, -400.0, 400.0],
                      [h, 30.0, -synth.SENSOR_HEIGHT, TUNNEL_TOP, -400.0, 400.0]])
    return synth.Scene(boxes, np.zeros((0, 4)), 400.0, TUNNEL_TOP)


def wall_and_ground():
    """One wall z in [3.5, 30] for |x| <= 400 and the ground; the sensor drives along x."""
    boxes = np.array([[-400.0, 400.0, -synth.SENSOR_HEIGHT, 6.0, TUNNEL_HALF_WIDTH, 30.0]])
    return synth.Scene(boxes, np.zeros((0, 4)), 400.0, 60.0)


WORLDS = {
    # name: (scene builder, body velocity, range noise sigma in metres).  The odometry fits its planes and lines to
    # 2 - 3 points of the last sweep: at synth's default 1 cm noise their normals tilt enough to observe the forward
    # translation (smallest eigenvalue ~75 in the tunnel), so these sensors are quieter.
    "tunnel": (tunnel, (0.0, 0.0, TUNNEL_SPEED), 2e-4),
    "wall": (wall_and_ground, (TUNNEL_SPEED, 0.0, 0.0), 0.0),
}
# odometry cases: world -> (sweep of the last clouds, start twist a few mrad and cm off, so that the loop takes several
# steps after iteration 0, eigenvalues of the first AtA below 10).  Mapping: the query sweep, the map's length, the
# start pose's offset from the true pose and the eigenvalues below 100 of the first AtA.
ODOM_CASES = {
    "tunnel": (0, np.array([0.004, -0.006, 0.003, 0.05, -0.04, 0.0], np.float32), 1),
    "wall": (0, np.array([0.01, -0.015, 0.008, 0.08, -0.06, 0.1], np.float32), 1),
}
MAP_SWEEP = 6
MAP_LENGTH = 60.0
MAP_OFFSET = np.array([0.004, 0.01, -0.005, 0.06, -0.05, 0.08], np.float32)
MAP_N_DEGENERATE = 1


def sweep(world, scene, lidar, k):
    """Sweep k of a world: constant velocity, no yaw, returns beyond MAX_RANGE dropped (ragged rings)."""
    _, v, noise = WORLDS[world]
    return synth.make_sweep(scene, lidar, k, scan_period=SCAN_PERIOD, v=v, yaw_rate=0.0, noise_sigma=noise,
                            max_range=MAX_RANGE)


def map_start(k=MAP_SWEEP):
    """Start pose of the scan-to-map loop on sweep k of the tunnel: the pose at the sweep's end, offset."""
    return (true_pose("tunnel", (k + 1) * SCAN_PERIOD) + MAP_OFFSET).astype(np.float32)


def true_pose(world, t):
    """Twist (rot x y z, pos x y z) of the sensor at time t."""
    v = np.asarray(WORLDS[world][1], np.float64)
    return np.concatenate([np.zeros(3), v * t]).astype(np.float32)


def tunnel_map(seed=7, length=MAP_LENGTH, surf_step=0.4, corner_step=0.2, jitter=0.02):
    """(corner M x 4, surf M x 4) float32: the walls, floor and ceiling on the surface lattice over |z| <= length / 2,
    corner points along the four wall / floor and wall / ceiling creases, +-jitter uniform as synth.make_map."""
    rng = np.random.RandomState(seed)
    h, y0, y1, z0 = TUNNEL_HALF_WIDTH, -synth.SENSOR_HEIGHT, TUNNEL_TOP, -length / 2
    ex, ey, ez = np.eye(3)
    surf = [synth._lattice_rect(np.array([-h, y0, z0]), ez, ey, length, y1 - y0, surf_step, rng, jitter),
            synth._lattice_rect(np.array([h, y0, z0]), ez, ey, length, y1 - y0, surf_step, rng, jitter),
            synth._lattice_rect(np.array([-h, y0, z0]), ex, ez, 2 * h, length, surf_step, rng, jitter),
            synth._lattice_rect(np.array([-h, y1, z0]), ex, ez, 2 * h, length, surf_step, rng, jitter)]
    corner = []
    zs = np.arange(z0 + corner_step / 2, -z0, corner_step)
    for cx in (-h, h):
        for cy in (y0, y1):
            c = np.stack([np.full_like(zs, cx), np.full_like(zs, cy), zs], axis=1)
            corner.append(c + rng.uniform(-jitter, jitter, size=c.shape))

    def pack(p):
        out = np.zeros((p.shape[0], 4), np.float32)
        out[:, :3] = p.astype(np.float32)
        return out
    return pack(np.concatenate(corner)), pack(np.concatenate(surf))


def odom_clouds(drv, world, scene, lidar, k0):
    """Restated registration of sweeps k0 and k0 + 1 -> (last corner, last surf, sharp, flat): the odometry's inputs
    with the last clouds' intensities floored (as transformToEnd leaves them)."""
    s = drv.scanreg()
    s.process(*sweep(world, scene, lidar, k0))
    last_c, last_s = s.cloud("less_sharp").copy(), s.cloud("less_flat").copy()
    last_c[:, 3] = np.floor(last_c[:, 3])
    last_s[:, 3] = np.floor(last_s[:, 3])
    s.process(*sweep(world, scene, lidar, k0 + 1))
    return last_c, last_s, s.cloud("sharp").copy(), s.cloud("flat").copy()


def map_queries(drv, world, scene, lidar, k):
    """The scan-to-map queries of sweep k: less sharp at the 0.2 m leaf, less flat at 0.4 m (restated)."""
    s = drv.scanreg()
    s.process(*sweep(world, scene, lidar, k))
    return drv.voxel_grid(s.cloud("less_sharp"), 0.2), drv.voxel_grid(s.cloud("less_flat"), 0.4)


def spectrum_margin(w, thr):
    """(eigenvalues below thr, largest below thr / thr, smallest at or above thr / thr) of ascending eigenvalues w."""
    w = np.sort(np.asarray(w, np.float64))
    lo, hi = w[w < thr], w[w >= thr]
    return lo.size, (lo.max() / thr if lo.size else 0.0), (hi.min() / thr if hi.size else math.inf)


# ---------------------------------------------------------------------------------------------- 6 x 6 spectra
LAMBDA_OVER_THR = (0.0, 1e-3, 0.5, 0.9, 0.99, 1.01, 1.1, 2.0, 10.0)
TRACES = (1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8)
PAIR_GAPS = (1e-1, 1e-2, 1e-3)


def random_orthogonal(rng):
    q, r = np.linalg.qr(rng.normal(size=(6, 6)))
    return q * np.sign(np.diag(r))[None, :]


def from_spectrum(lam, Q):
    """Q diag(lam) Q^T in float64, symmetrised, rounded to fp32."""
    A = (Q * np.asarray(lam, np.float64)[None, :]) @ Q.T
    return ((A + A.T) * 0.5).astype(np.float32)


def _fill(low, trace):
    """Six eigenvalues: `low` (the directions near or below thr) and the rest spread geometrically so that the sum is
    about `trace` (never below 20 thr, so they are clearly above it)."""
    n = 6 - len(low)
    rest = max(trace - sum(low), 1.0)
    hi = np.geomspace(1.0, 4.0, n)
    hi = hi / hi.sum() * rest
    return list(low) + list(hi)


def spectra(thr, seed=0):
    """Adversarial AtA around threshold thr -> list of (name, AtA fp32 6 x 6, AtB fp32 6).  Eigenvalues above thr are at
    least 20 thr; the trace runs from 1e1 to 1e8 (at the top the shortcut's 1e-5 tr margin exceeds thr)."""
    rng = np.random.RandomState(seed)
    out = []

    def add(name, lam):
        Q = random_orthogonal(rng)
        b = rng.normal(size=6) * np.sqrt(np.maximum(np.abs(lam), 1.0))
        out.append((name, from_spectrum(lam, Q), b.astype(np.float32)))

    for tr in TRACES:
        if tr < 30 * thr:
            continue
        for r in LAMBDA_OVER_THR:
            add(f"one:{r:g}:tr{tr:g}", _fill([r * thr], tr))
        for lows in ((0.3, 0.6), (0.5, 1.01), (0.1, 0.5, 0.9), (1e-3, 0.2, 0.99), (0.5, 2.0)):
            add(f"multi:{'/'.join(f'{v:g}' for v in lows)}:tr{tr:g}", _fill([v * thr for v in lows], tr))
        for gap in PAIR_GAPS:
            add(f"pair:{gap:g}:tr{tr:g}", _fill([0.5 * thr, 0.5 * thr * (1 + gap)], tr))
            add(f"triple:{gap:g}:tr{tr:g}", _fill([0.4 * thr, 0.4 * thr * (1 + gap), 0.4 * thr * (1 + 2 * gap)], tr))
    # exactly singular: the J of a scene that does not see one direction at all (two identical columns)
    J = rng.normal(size=(400, 6)) * np.array([3, 3, 3, 1, 1, 1])
    J[:, 5] = J[:, 3]
    A = (J.T @ J).astype(np.float32)
    out.append(("singular", A, (J.T @ rng.normal(size=400)).astype(np.float32)))
    # an exactly zero column and row
    J2 = J.copy()
    J2[:, 4] = 0.0
    out.append(("zero_column", (J2.T @ J2).astype(np.float32), (J2.T @ rng.normal(size=400)).astype(np.float32)))
    # a tiny negative eigenvalue, as the fp32 AtA of a rank-deficient J can have
    for tr in (1e3, 1e6):
        add(f"negative:tr{tr:g}", _fill([-1e-6 * tr, 0.5 * thr], tr))
    return out


def fp32_noise_band(AtA):
    """Half-width of the band around thr in which an fp32 eigen-decomposition of AtA cannot tell the side: 64 ulp of
    the largest eigenvalue (eps32 = 2^-23)."""
    w = np.linalg.eigvalsh(np.asarray(AtA, np.float64))
    return 64.0 * 2.0 ** -23 * float(np.abs(w).max())


def projection(AtA, drv, thr):
    """V^-1 V2 in float64 of the checker's fp32 eigenvectors (Eigen's solver, as the reference calls it): ROWS of V
    zeroed for the leading eigenvalues below thr -> (P 6 x 6 float64, degenerate)."""
    w, V = drv.eig_sym(np.asarray(AtA, np.float32))
    V = V.astype(np.float64)
    V2 = V.copy()
    deg = False
    for i in range(6):
        if w[i] < thr:
            V2[i, :] = 0.0
            deg = True
        else:
            break
    return np.linalg.inv(V) @ V2, deg


# ---------------------------------------------------------------------------------------------- loop replay
VARIANTS = ("carried", "first_only", "none", "identity", "rebuilt")


def _deltas(x):
    """rad2deg / x100 convergence measures (BasicLaserOdometry.cpp:614-621): float rad2deg, double sum, float sqrt."""
    dr = math.sqrt(sum(float(F(float(v) * 180.0 / math.pi)) ** 2 for v in x[:3]))
    dt = math.sqrt(sum(float(F(v) * F(100)) ** 2 for v in x[3:]))
    return F(dr), F(dt)


def replay(normal_eq, start, drv, thr, min_sel, max_iter, delta, variant="carried"):
    """The Gauss-Newton loop with the checker's plain solve (qr_solve6) and a float64 projection -> (twist fp32,
    iterations, degenerate, per-iteration log).  normal_eq(it, twist) returns (AtA, AtB, n_selected) at the replay's
    pose.  variant: "carried" is the upstream rule; the others are wrong on purpose --
      first_only: P applied on iteration 0 only; none: never projected; identity: P = V^-1 V (no row zeroed);
      rebuilt: P recomputed from every iteration's AtA."""
    t = np.array(start, np.float32).reshape(6)
    P, deg, iters, log = None, False, 0, []
    for it in range(max_iter):
        iters = it + 1
        AtA, AtB, n_sel = normal_eq(it, t)
        if n_sel < min_sel:
            log.append((it, n_sel, None))
            continue
        x = drv.qr_solve6(AtA, AtB).astype(np.float64)
        if it == 0 or variant == "rebuilt":
            P, deg_now = projection(AtA, drv, thr)
            if it == 0:
                deg = deg_now
            if variant == "identity":
                w, V = drv.eig_sym(np.asarray(AtA, np.float32))
                P = np.linalg.inv(V.astype(np.float64)) @ V.astype(np.float64)
            if variant == "rebuilt" and not deg_now:
                P = None
        use = deg and P is not None and (variant != "none") and (variant != "first_only" or it == 0)
        if use:
            x = P @ x
        x = x.astype(np.float32)
        t = (t + x).astype(np.float32)
        log.append((it, n_sel, x))
        dr, dt = _deltas(x)
        if dr < F(delta) and dt < F(delta):
            break
    return t, iters, deg, log
