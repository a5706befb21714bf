"""numpy restatement of the alignment against the whole-run voxel map (csrc/densemap.cuh: dense_align_kernel;
csrc/stages.inc: loam_b200_dense_align; include/loam_b200.h "Alignment against the whole-run voxel map").

The target is what dense_reference / normals_reference export: ascending keys, fp32 centroids and normals.  Every
floating-point operation of an iteration is the kernel's, in the kernel's order (fp32, no FMA):
  * q = pointAssociateToMap(pose, p) (map_reference.Pose.to_map); a non-finite p has no correspondence;
  * v = q's voxel (dense_reference.voxel_keys at the target's leaf); outside the key range: no correspondence;
  * candidates: the voxels within `radius` of v on every axis (an offset outside the key range does not exist) whose
    normal_x is not NaN, in ascending key order (normals_reference.offsets); d = c - q, d2 = (dx*dx + dy*dy) + dz*dz;
    the first candidate with d2 below every earlier one and below the gate wins (strict <); gate = s * s in fp32 with
    s = (float)radius * leaf;
  * pd2 = (nx*(qx - cx) + ny*(qy - cy)) + nz*(qz - cz); s = 1 - 0.9f*|pd2| / sqrtf(sqrtf((px*px + py*py) + pz*pz)) with
    the sensor-frame p; selected when (double)s > 0.1; coeff = s * (nx, ny, nz, pd2);
  * Jacobian row of the scan-to-map kernels (map_args_from's products) and rhs = -coeff.w;
  * 29 sums per point (21 AtA, 6 AtB, 1, pd2^2; zeros when not selected) -> per warp of 32 points the fp32 xor
    butterfly (lane l adds lane l ^ o for o = 16, 8, 4, 2, 1), per CTA of 128 points the 4 warp sums added to 0.0f in
    warp order, then the CTA partials in double: group w (0..3) adds CTAs w, w + 4, ... to 0.0 in order, the 4 group
    sums are added to 0.0 in order, and the total is rounded to fp32.
The loop follows the mapping stage's policy with api.gn_solve (the library's host solve) and float pose updates.
"""
import math

import numpy as np

import dense_reference as dr
import map_reference as mr
import normals_reference as nr
from loam_velodyne_b200.api import gn_solve

F = np.float32
HALF = dr.HALF
NEQ = 32
LM_THREADS = 128


class Target:
    def __init__(self, leaf, keys, cent, nrm):
        self.leaf = F(leaf)
        self.keys = np.asarray(keys, np.uint64)
        self.cent = np.ascontiguousarray(cent, np.float32).reshape(-1, 4)
        self.nrm = np.ascontiguousarray(nrm, np.float32).reshape(-1, 4)


def built_target(ref, radius, viewpoint, drv, keep=None):
    """The target loam_b200_dense_target_build makes of a DenseMapRef (keep: the miss-ratio filter's mask)."""
    cent, _ = ref.export()
    keys = ref.keys
    if keep is not None:
        cent, keys = cent[keep], keys[keep]
    return Target(ref.leaf, keys, cent, nr.normals(keys, cent, radius, viewpoint, drv))


def loaded_target(leaf, cent, nrm):
    """The target loam_b200_dense_target_load makes of host entries; ValueError where the library says ERR_ARG."""
    cent = np.ascontiguousarray(cent, np.float32).reshape(-1, 4)
    keys = dr.voxel_keys(cent, leaf)
    if (keys == dr.EMPTY).any():
        raise ValueError("a centroid is not finite or its voxel is outside the key range")
    o = np.argsort(keys, kind="stable")
    if (keys[o][1:] == keys[o][:-1]).any():
        raise ValueError("two entries lie in the same voxel")
    return Target(leaf, keys[o], cent[o], np.asarray(nrm, np.float32).reshape(-1, 4)[o])


def gate(radius, leaf):
    s = F(F(radius) * F(leaf))
    return F(s * s)


def map_args(pose):
    """(A, B, C) of map_args_from (csrc/mapping_lm.cuh) from a map_reference.Pose, products left to right in fp32."""
    srx, sry, srz = pose.s
    crx, cry, crz = pose.c
    z = F(0.0)
    A = [crx * sry * srz, crx * crz * sry, -(srx * sry), -srx * srz, -(crz * srx), -crx, crx * cry * srz,
         crx * cry * crz, -(cry * srx)]
    B = [cry * srx * srz - crz * sry, sry * srz + cry * crz * srx, crx * cry, z, z, z, -cry * crz - srx * sry * srz,
         cry * srz - crz * srx * sry, -(crx * sry)]
    C = [crz * srx * sry - cry * srz, -cry * crz - srx * sry * srz, z, crx * crz, -(crx * srz), z,
         sry * srz + cry * crz * srx, crz * sry - cry * srx * srz, z]
    return [F(v) for v in A], [F(v) for v in B], [F(v) for v in C]


def search(target, q, radius, gate_le=False, tie_le=False, any_normal=False, wrap=False, clamp=False):
    """Index of the accepted match per map-frame point q (N x 4), -1 when none.  The keyword arguments are the
    deliberately wrong variants of the sensitivity tests: <= at the gate, <= between candidates (the last of a tie
    wins), candidates without a normal, key + offset arithmetic that wraps rows, and a voxel outside the key range
    clamped into it instead of having no correspondence."""
    n = q.shape[0]
    best = np.full(n, -1, np.int64)
    m = target.keys.size
    if m == 0 or n == 0:
        return best
    g = gate(radius, target.leaf)
    best_d2 = np.full(n, g, np.float32)
    if clamp:
        inv = F(1.0) / target.leaf
        with np.errstate(invalid="ignore", over="ignore"):
            f = np.floor(q[:, :3] * inv)
        ok_q = np.isfinite(f).all(axis=1)
        vox = np.clip(np.where(ok_q[:, None], f, 0.0), -HALF, HALF - 1).astype(np.int64)
        vkey = np.where(ok_q, nr.pack(vox), dr.EMPTY)
    else:
        vkey = dr.voxel_keys(q, target.leaf)
        ok_q = vkey != dr.EMPTY
        vox = dr.key_voxel(np.where(ok_q, vkey, np.uint64(0)))
    has_n = np.ones(m, bool) if any_normal else ~np.isnan(target.nrm[:, 0])
    first = np.ones(n, bool)
    for off in nr.offsets(radius):
        wk, ok = (nr.naive_neighbour if wrap else nr.neighbour)(vkey, vox, off)
        pos = np.minimum(np.searchsorted(target.keys, wk), m - 1)
        found = ok_q & ok & (target.keys[pos] == wk) & has_n[pos]
        c = target.cent[pos]
        dx, dy, dz = c[:, 0] - q[:, 0], c[:, 1] - q[:, 1], c[:, 2] - q[:, 2]
        d2 = (dx * dx + dy * dy) + dz * dz
        le = np.where(first, gate_le, tie_le)
        better = found & ((d2 < best_d2) | (le & (d2 == best_d2)))
        first &= ~better
        best = np.where(better, pos, best)
        best_d2 = np.where(better, d2, best_d2)
    return best


def search_brute(target, q, radius):
    """The same over every target voxel (fp32, key order, first smallest wins, d2 < gate), in chunks."""
    g = gate(radius, target.leaf)
    c = target.cent[:, :3]
    has_n = ~np.isnan(target.nrm[:, 0])
    out = np.full(q.shape[0], -1, np.int64)
    if c.shape[0] == 0:
        return out
    for s in range(0, q.shape[0], 256):
        qq = q[s:s + 256, :3]
        dx = c[None, :, 0] - qq[:, None, 0]
        dy = c[None, :, 1] - qq[:, None, 1]
        dz = c[None, :, 2] - qq[:, None, 2]
        d2 = (dx * dx + dy * dy) + dz * dz
        d2[:, ~has_n] = np.inf
        with np.errstate(invalid="ignore"):
            d2[~np.isfinite(qq).all(axis=1)] = np.inf
        j = np.argmin(d2, axis=1)
        out[s:s + 256] = np.where(d2[np.arange(j.size), j] < g, j, -1)
    return out


def iterate(target, pts, twist6, radius, map_frame_weight=False, nonfinite_as_origin=False, **variant):
    """One iteration -> (32 fp32 sums, match N, coeff N x 4, selected N bool).  map_frame_weight and
    nonfinite_as_origin are deliberately wrong variants of the sensitivity tests (the mapping stage's range of q instead
    of p; a non-finite point taken as the sensor origin), the other keywords those of search()."""
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
    n = p.shape[0]
    pose = mr.Pose(twist6)
    finite = np.isfinite(p[:, :3]).all(axis=1)
    p_used = np.where(finite[:, None], p, F(0.0)) if nonfinite_as_origin else p
    with np.errstate(invalid="ignore", over="ignore"):
        q = pose.to_map(np.where(finite[:, None], p, F(0.0)))
    if not nonfinite_as_origin:
        q[~finite] = np.nan
    p = p_used
    match = search(target, q, radius, **variant)
    has = match >= 0
    coeff = np.zeros((n, 4), np.float32)
    sel = np.zeros(n, bool)
    acc = np.zeros((n, 29), np.float32)
    if has.any():
        j = match[has]
        c, nv, qh, ph = target.cent[j], target.nrm[j], q[has], p[has]
        pd2 = (nv[:, 0] * (qh[:, 0] - c[:, 0]) + nv[:, 1] * (qh[:, 1] - c[:, 1])) + nv[:, 2] * (qh[:, 2] - c[:, 2])
        r = qh if map_frame_weight else ph
        with np.errstate(divide="ignore", invalid="ignore"):
            s = F(1.0) - F(0.9) * np.abs(pd2) / np.sqrt(np.sqrt((r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1]) + r[:, 2] * r[:, 2]))
            cf = np.stack([s * nv[:, 0], s * nv[:, 1], s * nv[:, 2], s * pd2], axis=1)
        coeff[has] = cf
        sh = s.astype(np.float64) > 0.1
        sel[np.nonzero(has)[0][sh]] = True
        rows, rhs = jacobian_rows(pose, ph[sh], cf[sh])
        a = np.zeros((rows.shape[0], 29), np.float32)
        k = 0
        for i in range(6):
            for t in range(i, 6):
                a[:, k] = rows[:, i] * rows[:, t]
                k += 1
        for i in range(6):
            a[:, 21 + i] = rows[:, i] * rhs
        a[:, 27] = F(1.0)
        a[:, 28] = pd2[sh] * pd2[sh]
        acc[np.nonzero(has)[0][sh]] = a
    return reduce_sums(acc), match, coeff, sel


def jacobian_rows(pose, po, coeff):
    A, B, C = map_args(pose)
    px, py, pz = po[:, 0], po[:, 1], po[:, 2]
    cx, cy, cz, cw = coeff[:, 0], coeff[:, 1], coeff[:, 2], coeff[:, 3]
    r0 = ((A[0] * px + A[1] * py + A[2] * pz) * cx + (A[3] * px + A[4] * py + A[5] * pz) * cy +
          (A[6] * px + A[7] * py + A[8] * pz) * cz)
    r1 = (B[0] * px + B[1] * py + B[2] * pz) * cx + (B[6] * px + B[7] * py + B[8] * pz) * cz
    r2 = (C[0] * px + C[1] * py) * cx + (C[3] * px + C[4] * py) * cy + (C[6] * px + C[7] * py) * cz
    return np.stack([r0, r1, r2, cx, cy, cz], axis=1).astype(np.float32), -cw


def reduce_sums(acc):
    """29 per-point sums (N x 29 fp32) -> the 32 fp32 results of reduce_normal_equations."""
    n = acc.shape[0]
    out = np.zeros(NEQ, np.float32)
    if n == 0:
        return out
    nb = -(-n // LM_THREADS)
    v = np.zeros((nb * LM_THREADS, 29), np.float32)
    v[:n] = acc
    v = v.reshape(nb, 4, 32, 29)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[:, :, lanes ^ o, :]
    w = v[:, :, 0, :]
    part = np.zeros((nb, NEQ), np.float32)
    for k in range(4):
        part[:, :29] = part[:, :29] + w[:, k, :]
    tot = np.zeros(NEQ, np.float64)
    for g in range(4):
        s = np.zeros(NEQ, np.float64)
        for b in range(g, nb, 4):
            s = s + part[b].astype(np.float64)
        tot = tot + s
    return tot.astype(np.float32)


def normal_eq(r):
    """32 sums -> (AtA 6 x 6, AtB 6, n_selected, sum of pd2^2) as the library unpacks them."""
    AtA = np.zeros((6, 6), np.float32)
    k = 0
    for i in range(6):
        for j in range(i, 6):
            AtA[i, j] = AtA[j, i] = r[k]
            k += 1
    n_sel = int(r[27] + F(0.5)) if np.isfinite(r[27]) else 0
    return AtA, r[21:27].copy(), n_sel, r[28]


def rad2deg(r):
    return F(float(r) * 180.0 / math.pi)


def converged(x):
    """BasicLaserMapping.cpp:420-422: std::pow of a float promotes to double, the sqrt is stored in a float."""
    dr_ = F(math.sqrt(float(rad2deg(x[0])) ** 2 + float(rad2deg(x[1])) ** 2 + float(rad2deg(x[2])) ** 2))
    dt = F(math.sqrt(float(F(x[3] * F(100))) ** 2 + float(F(x[4] * F(100))) ** 2 + float(F(x[5] * F(100))) ** 2))
    return dr_ < F(0.05) and dt < F(0.05)


def projection(AtA, drv, thr=100.0):
    """The degeneracy projection V^-1 V2 in float64 as tests/test_abi.py states it: the checker's eigenvectors (Eigen's
    solver, whose signs the library's sym_eigen<6> shares), ROWS zeroed for the leading eigenvalues below thr."""
    w, V = drv.eig_sym(np.asarray(AtA, np.float32))
    V = V.astype(np.float64)
    V2 = V.copy()
    for i in range(6):
        if w[i] < thr:
            V2[i, :] = 0.0
        else:
            break
    return np.linalg.inv(V) @ V2


def align(target, pts, twist6, radius, max_iterations, step=None, drv=None):
    """The loop of loam_b200_dense_align -> (twist6 fp32, info dict as api.Ctx.dense_align).  step(twist) may replace
    the restated iteration (the GPU replay passes Ctx.dense_align_iterate).  Once the first solve reports degenerate,
    later steps apply projection() of that iteration's AtA (drv: the checker) to the plain solve: equal to the library
    within 2e-4."""
    t = np.array(twist6, np.float32).reshape(6)
    info = {"iterations": 0, "n_selected": 0, "rms": F(0.0), "degenerate": False, "converged": False}
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
    if p.shape[0] == 0 or target.keys.size == 0:
        return t, info
    solved, P = False, None
    for it in range(max_iterations):
        r = step(t) if step is not None else iterate(target, p, t, radius)[0]
        AtA, AtB, n_sel, ss = normal_eq(r)
        info["iterations"] = it + 1
        info["n_selected"] = n_sel
        info["rms"] = F(math.sqrt(float(ss) / n_sel)) if n_sel > 0 else F(0.0)
        if n_sel < 50:
            continue
        if not solved:
            x, deg = gn_solve(AtA, AtB, True, 100.0)
            info["degenerate"] = deg
            P = projection(AtA, drv) if deg else None
            solved = True
        else:
            x, _ = gn_solve(AtA, AtB, False, 100.0)
            if P is not None:
                x = (P @ x.astype(np.float64)).astype(np.float32)
        t = (t + x.astype(np.float32)).astype(np.float32)
        if converged(x):
            info["converged"] = True
            break
    return t, info


# ---- hand-made cases
EDGE_LEAF = 0.5  # 1 / leaf is exact; every coordinate below is exact in fp32
NAN = np.float32(np.nan)


def edge_cases():
    """{name: (centroids M x 4, normals M x 4, points N x 4 (sensor frame), twist6, radius, variants)}, where each
    variant (keyword arguments of iterate()) is a deliberately wrong restatement that changes the result on that case;
    None for the empty target, on which nothing can differ."""
    h = EDGE_LEAF
    zero = (0.0, 0.0, 0.0, 0.0, 0.0, 0.0)
    cases = {}
    # two centroids at exactly the same d2 = 0.0625 from q with different normals: the first in key order wins
    cases["tie"] = ([(10.0, 0.25, 0.25, 1.0), (10.5, 0.25, 0.25, 1.0)], [(1, 0, 0, 0), (0, 1, 0, 0)],
                    [(10.25, 0.25, 0.25, 0.0)], zero, 1, [{"tie_le": True}])
    # d2 exactly at the gate (0.25 at radius 1): rejected
    cases["gate"] = ([(0.75, 0.25, 0.25, 1.0)], [(0, 0, 1, 0)], [(0.25, 0.25, 0.25, 0.0)], zero, 1,
                     [{"gate_le": True}])
    # the nearest voxel has no normal, a farther one has
    cases["no_normal"] = ([(3.125, 1.25, 1.25, 1.0), (3.875, 1.25, 1.25, 1.0)], [(NAN, NAN, NAN, NAN), (0, 1, 0, 0.1)],
                          [(3.25, 1.25, 1.25, 0.0)], zero, 2, [{"any_normal": True}])
    # key-range edges: a point just beyond the last x voxel (no correspondence, though a centroid is 0.1875 m away),
    # and a point in the last x voxel of a row beside the first voxel of the next row (never a candidate)
    e = F(HALF * h)
    cases["key_range"] = ([(e - F(0.125), 0.25, 0.25, 1.0), (-e + F(0.25), 0.75, 0.25, 1.0)],
                          [(1, 0, 0, 0), (0, 0, 1, 0)], [(e + F(0.0625), 0.25, 0.25, 0.0), (e - F(0.25), 0.25, 0.25, 0.0)],
                          zero, 1, [{"clamp": True}])
    # the weight's range: the sensor is 100 m from the map origin, the point 4 m from the sensor
    cases["sensor_range"] = ([(104.25, 0.25, 0.25, 1.0)], [(1, 0, 0, 0)], [(4.125, 0.25, 0.25, 0.0)],
                             (0.0, 0.0, 0.0, 100.0, 0.0, 0.0), 1, [{"map_frame_weight": True}])
    # non-finite points, with a centroid beside the sensor position
    cases["non_finite"] = ([(0.25, 0.25, 0.25, 1.0)], [(0, 1, 0, 0)],
                           [(NAN, 0.0, 0.0, 0.0), (np.inf, 1.0, 1.0, 0.0), (0.0, -np.inf, 0.0, 0.0)], zero, 1,
                           [{"nonfinite_as_origin": True}])
    cases["empty"] = ([], [], [(1.0, 2.0, 3.0, 0.0)], zero, 3, None)
    out = {}
    for k, (c, nrm, p, tw, r, var) in cases.items():
        out[k] = (np.array(c, np.float32).reshape(-1, 4), np.array(nrm, np.float32).reshape(-1, 4),
                  np.array(p, np.float32).reshape(-1, 4), np.array(tw, np.float32), r, var)
    return out


def plane_case(n=4000, seed=5):
    """One plane: the ground y = -1.75 under the sensor, centroids on a 0.5 m grid with normal +y, and sensor-frame
    points on it -> (centroids, normals, points).  Only y, rot_x and rot_z are observable."""
    g = np.arange(-40, 40) * EDGE_LEAF + F(0.25)
    X, Z = np.meshgrid(g, g)
    c = np.stack([X.ravel(), np.full(X.size, -1.75), Z.ravel(), np.ones(X.size)], axis=1).astype(np.float32)
    nrm = np.tile(np.array([0, 1, 0, 0], np.float32), (c.shape[0], 1))
    rng = np.random.RandomState(seed)
    xz = rng.uniform(-15, 15, (n, 2))
    p = np.stack([xz[:, 0], np.full(n, -1.75), xz[:, 1], np.zeros(n)], axis=1).astype(np.float32)
    return c, nrm, p


# ---- static sweeps ray-cast from known poses (no motion during the sweep)
def to_map64(twist6, v):
    """rotateZXY then translate in float64: the map-frame position of sensor-frame vectors v (N x 3)."""
    rx, ry, rz = (float(a) for a in twist6[:3])
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    x1 = math.cos(rz) * x - math.sin(rz) * y
    y1 = math.sin(rz) * x + math.cos(rz) * y
    y2 = math.cos(rx) * y1 - math.sin(rx) * z
    z2 = math.sin(rx) * y1 + math.cos(rx) * z
    x3 = math.cos(ry) * x1 + math.sin(ry) * z2
    z3 = math.cos(ry) * z2 - math.sin(ry) * x1
    return np.stack([x3, y2, z3], axis=1)


def static_sweep(scene, lidar, twist6, seed, noise_sigma=0.005):
    """-> (sensor-frame points N x 4 float32, the same in the map frame) of a sweep taken at rest at twist6."""
    from loam_velodyne_b200 import synth
    R, A = lidar.n_rings, lidar.n_az
    elev = np.radians(np.linspace(lidar.lower_deg, lidar.upper_deg, R))
    theta = 2.0 * math.pi * np.arange(A) / A
    ce, se = np.cos(elev)[:, None], np.sin(elev)[:, None]
    dl = np.stack([-np.sin(theta)[None, :] * ce, np.broadcast_to(se, (R, A)), np.cos(theta)[None, :] * ce],
                  axis=-1).reshape(-1, 3)
    o = np.broadcast_to(np.asarray(twist6[3:], np.float64), dl.shape)
    t = synth._raycast(scene, np.ascontiguousarray(o), to_map64(twist6, dl))
    t = t + np.random.RandomState(seed).normal(0.0, noise_sigma, t.shape)
    ok = np.isfinite(t) & (t > 0.5)
    ring = np.repeat(np.arange(R, dtype=np.float32), A)
    sensor = np.concatenate([(t[ok, None] * dl[ok]).astype(np.float32), ring[ok, None]], axis=1)
    world = np.concatenate([(to_map64(twist6, t[ok, None] * dl[ok]) + o[ok]).astype(np.float32), ring[ok, None]],
                           axis=1)
    return np.ascontiguousarray(sensor), np.ascontiguousarray(world)


def twist_error(a, b):
    """(translation error in metres, rotation error in degrees: the angle of R(a)^T R(b))."""
    e = np.eye(3)
    Ra, Rb = to_map64(a, e).T, to_map64(b, e).T
    c = (np.trace(Ra.T @ Rb) - 1.0) / 2.0
    return float(np.linalg.norm(np.asarray(a[3:], np.float64) - np.asarray(b[3:], np.float64))), \
        math.degrees(math.acos(min(1.0, max(-1.0, c))))


def perturbations(seed, n, metres=0.3, degrees=2.0):
    """n twists of ~`metres` and ~`degrees`: random directions, exact magnitudes."""
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        u = rng.normal(size=3)
        w = rng.normal(size=3)
        out.append(np.concatenate([w / np.linalg.norm(w) * math.radians(degrees), u / np.linalg.norm(u) * metres]))
    return out
