"""numpy restatement of the ray cast into the whole-run voxel map's target (csrc/densemap.cuh: dense_raycast_kernel;
include/loam_b200.h "Ray casting the whole-run voxel map").

The target is align_reference.Target (ascending keys, fp32 centroids and normals).  Every floating-point operation is
the kernel's, in the kernel's order, fp64 without FMA:
  * |p| = sqrt((x*x + y*y) + z*z) of the float components, u = p / |p|; a non-finite or zero p has no hit;
  * d = rotZ, rotX, rotY of u (align_reference.to_map64's formula) with math.cos / math.sin (the C library's, as the
    host's std::cos / std::sin) of the pose's float angles; o = the pose's float position;
  * start voxel floor(o_a / L), L = (double)leaf; t_next_a = ((double)k * L - o_a) * (1.0 / d_a), k = v_a + 1 when
    d_a > 0, v_a when d_a < 0, +inf when d_a == 0;
  * per voxel [t_enter, t_exit = min t_next): stop when t_enter > max_range; hit the first occupied voxel with
    t_exit > min_range; else step along the smallest t_next (ties x, y, z), t_enter = its old t_next, recompute it;
  * hit: lo = max(t_enter, min_range), hi = t_exit; t = clamp(num / den, lo, hi) on the voxel's surfel when it has a
    normal and den != 0, else lo; t > max_range is no hit.  range = (float)t, index = position in the target.
Vectorised over rays, one loop iteration per step; voxels are looked up with np.searchsorted on the target's keys (the
restatement has no bricks: the GPU's brick index must not change a bit).
"""
import math

import numpy as np

HALF = 1 << 20
MAX_STEPS = 3 * 65536 + 4  # max_range / leaf <= 65536 crosses at most sqrt(3) 65536 + 3 faces


def trig(twist6):
    """(cx, sx, cy, sy, cz, sz): cos / sin in double of the pose's float rot_x, rot_y, rot_z."""
    t = np.asarray(twist6, np.float32).reshape(6)
    out = []
    for a in range(3):
        r = float(t[a])
        out += [math.cos(r), math.sin(r)]
    return out


def directions(rays, twist6, zero_eps=False):
    """-> (map-frame unit directions N x 3 float64, valid N bool).  zero_eps: a deliberately wrong variant that takes a
    tiny ray (|p| < 1e-6) as zero."""
    p = np.ascontiguousarray(rays, np.float32).reshape(-1, 4)
    x, y, z = (p[:, a].astype(np.float64) for a in range(3))
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        ln = np.sqrt((x * x + y * y) + z * z)
        ok = np.isfinite(p[:, :3]).all(axis=1) & (ln > 0.0)
        if zero_eps:
            ok &= ln >= 1e-6
        ux, uy, uz = x / ln, y / ln, z / ln
    cx, sx, cy, sy, cz, sz = trig(twist6)
    x1 = cz * ux - sz * uy
    y1 = sz * ux + cz * uy
    y2 = cx * y1 - sx * uz
    z2 = sx * y1 + cx * uz
    d = np.stack([cy * x1 + sy * z2, y2, cy * z2 - sy * x1], axis=1)
    return d, ok


def lookup(target, v, wrap=False):
    """Target index of the voxels v (M x 3 int64), -1 when not occupied.  wrap: a deliberately wrong variant whose
    key arithmetic carries an index outside the key range into the next row."""
    u = v + HALF
    if wrap:
        valid = (u >= 0).all(axis=1)
        key = (u[:, 2] << 42) + (u[:, 1] << 21) + u[:, 0]
    else:
        valid = ((v >= -HALF) & (v < HALF)).all(axis=1)
        key = (u[:, 2] << 42) | (u[:, 1] << 21) | u[:, 0]
    m = target.keys.size
    k = np.where(valid, key, 0).astype(np.uint64)
    pos = np.minimum(np.searchsorted(target.keys, k), m - 1)
    return np.where(valid & (target.keys[pos] == k), pos, -1)


def cast(target, rays, twist6, min_range=0.0, max_range=100.0, max_steps=MAX_STEPS, tie_z_first=False, trunc=False,
         zero_inv=False, exit_ge=False, min_ignored=False, no_clamp=False, no_normal_exit=False,
         den_zero_divide=False, max_ge=False, no_t_max=False, wrap=False, zero_eps=False):
    """-> (range float32[N], index int32[N]).  The keyword arguments after max_steps are deliberately wrong variants of
    the sensitivity tests: ties to z first, a truncated start voxel, the t_next formula on an axis with d == 0,
    t_exit >= min_range, no min_range test, no clamp to the segment, the exit instead of the entry without a normal,
    num / den taken at den == 0, t >= max_range as no hit, no max_range test at the hit, wrapping keys, tiny rays as
    zero."""
    p = np.ascontiguousarray(rays, np.float32).reshape(-1, 4)
    n = p.shape[0]
    rng = np.full(n, np.inf, np.float32)
    idx = np.full(n, -1, np.int32)
    if n == 0 or target.keys.size == 0:
        return rng, idx
    tw = np.asarray(twist6, np.float32).reshape(6)
    d, ok = directions(p, tw, zero_eps)
    rows = np.nonzero(ok)[0]
    d = d[rows]
    m = rows.size
    o = np.array([float(tw[3]), float(tw[4]), float(tw[5])])
    L = float(np.float32(target.leaf))
    mn, mx = float(np.float32(min_range)), float(np.float32(max_range))
    start = (np.trunc if trunc else np.floor)(o / L).astype(np.int64)
    v = np.tile(start, (m, 1))
    with np.errstate(divide="ignore"):
        inv = 1.0 / d
    tn = np.empty((m, 3))
    with np.errstate(invalid="ignore"):
        for a in range(3):
            k = np.where(d[:, a] > 0.0, v[:, a] + 1, v[:, a])
            t = (k.astype(np.float64) * L - o[a]) * inv[:, a]
            tn[:, a] = t if zero_inv else np.where(d[:, a] != 0.0, t, np.inf)
    t_enter = np.zeros(m)
    hit_j = np.full(m, -1, np.int64)
    lo = np.zeros(m)
    hi = np.zeros(m)
    act = np.arange(m)
    for _ in range(max_steps):
        te = t_enter[act]
        go = ~(te > mx)
        act, te = act[go], te[go]
        if act.size == 0:
            break
        x, y, z = tn[act, 0], tn[act, 1], tn[act, 2]
        if tie_z_first:
            ax = np.where((z <= y) & (z <= x), 2, np.where(y <= x, 1, 0))
        else:
            ax = np.where((x <= y) & (x <= z), 0, np.where(y <= z, 1, 2))
        tx = tn[act, ax]
        j = lookup(target, v[act], wrap)
        past = np.ones(act.size, bool) if min_ignored else ((tx >= mn) if exit_ge else (tx > mn))
        h = (j >= 0) & past
        if h.any():
            a = act[h]
            hit_j[a] = j[h]
            lo[a] = np.where(te[h] > mn, te[h], mn)
            hi[a] = tx[h]
        act, ax, tx = act[~h], ax[~h], tx[~h]
        t_enter[act] = tx
        fwd = d[act, ax] > 0.0
        v[act, ax] += np.where(fwd, 1, -1)
        k = np.where(fwd, v[act, ax] + 1, v[act, ax])
        with np.errstate(invalid="ignore"):
            tn[act, ax] = (k.astype(np.float64) * L - o[ax]) * inv[act, ax]
    hj = np.nonzero(hit_j >= 0)[0]
    if hj.size == 0:
        return rng, idx
    j = hit_j[hj]
    l, h, dd = lo[hj], hi[hj], d[hj]
    nv = target.nrm[j].astype(np.float64)
    c = target.cent[j].astype(np.float64)
    has_n = ~np.isnan(target.nrm[j, 0])
    with np.errstate(invalid="ignore", divide="ignore"):
        den = (nv[:, 0] * dd[:, 0] + nv[:, 1] * dd[:, 1]) + nv[:, 2] * dd[:, 2]
        num = (nv[:, 0] * (c[:, 0] - o[0]) + nv[:, 1] * (c[:, 1] - o[1])) + nv[:, 2] * (c[:, 2] - o[2])
        q = num / den
    use = has_n & ((den != 0.0) | den_zero_divide)
    clamped = q if no_clamp else np.where(q < l, l, np.where(q > h, h, q))
    t = np.where(use, clamped, np.where(~has_n, h, l) if no_normal_exit else l)
    if no_t_max:
        stop = np.zeros(t.size, bool)
    else:
        stop = (t >= mx) if max_ge else (t > mx)
    keep = hj[~stop]
    rng[rows[keep]] = t[~stop].astype(np.float32)
    idx[rows[keep]] = j[~stop]
    return rng, idx


def cast_brute(target, rays, twist6, min_range=0.0):
    """The first crossed occupied voxel by slab test over every target voxel, without a max range -> (index N, entry
    N, gap N): a voxel is crossed when its slab exit is beyond max(slab entry, 0) and beyond min_range; the hit is the
    smallest entry; gap is the distance to the next-smallest entry (to exclude rays through edges and corners)."""
    tw = np.asarray(twist6, np.float32).reshape(6)
    d, ok = directions(rays, tw)
    o = np.array([float(tw[3]), float(tw[4]), float(tw[5])])
    L = float(np.float32(target.leaf))
    mn = float(np.float32(min_range))
    k = target.keys.astype(np.int64)
    vox = np.stack([k & (2 * HALF - 1), (k >> 21) & (2 * HALF - 1), k >> 42], axis=1) - HALF
    lo_b = vox.astype(np.float64) * L
    hi_b = (vox + 1).astype(np.float64) * L
    n = d.shape[0]
    out = np.full(n, -1, np.int64)
    entry = np.full(n, np.inf)
    gap = np.full(n, np.inf)
    for i in np.nonzero(ok)[0]:
        with np.errstate(divide="ignore", invalid="ignore"):
            inv = 1.0 / d[i]
            t1 = (lo_b - o) * inv
            t2 = (hi_b - o) * inv
        par = d[i] == 0.0
        inside = (lo_b <= o) & (o < hi_b)
        t1 = np.where(par, np.where(inside, -np.inf, np.inf), t1)
        t2 = np.where(par, np.where(inside, np.inf, -np.inf), t2)
        tn = np.minimum(t1, t2).max(axis=1)
        tf = np.maximum(t1, t2).min(axis=1)
        en = np.maximum(tn, 0.0)
        crossed = (tf > en) & (tf > mn)
        if not crossed.any():
            continue
        e = np.where(crossed, en, np.inf)
        o2 = np.argsort(e, kind="stable")
        out[i] = o2[0]
        entry[i] = e[o2[0]]
        gap[i] = e[o2[1]] - e[o2[0]] if e.size > 1 else np.inf
    return out, entry, gap


# ---- hand-made cases
LEAF = 0.5  # every coordinate below is exact in fp32; 1 / leaf is exact
NAN = np.float32(np.nan)


def _centre(i, j, k):
    return ((i + 0.5) * LEAF, (j + 0.5) * LEAF, (k + 0.5) * LEAF)


def edge_cases():
    """{name: (centroids M x 4, normals M x 4, rays N x 4, twist6, min_range, max_range, expected voxels, variants)}:
    expected[i] is the voxel (i, j, k) ray i hits, or None; each variant (keyword arguments of cast()) is a deliberately
    wrong restatement that changes the result on that case."""
    no = (NAN, NAN, NAN, NAN)
    at = (0.0, 0.0, 0.0, 0.25, 0.25, 0.25)  # inside voxel (0, 0, 0)
    cases = {}

    def vox(ijk, nrm=no, cent=None):
        c = _centre(*ijk) if cent is None else cent
        return (c[0], c[1], c[2], 1.0), nrm

    def case(name, voxels, rays, twist, mn, mx, expect, variants):
        cases[name] = ([v[0] for v in voxels], [v[1] for v in voxels], rays, twist, mn, mx, expect, variants)

    # d_y = d_z = 0: t_next is +inf on those axes (the formula there would walk -y forever)
    case("axis_parallel", [vox((3, 0, 0))], [(2.0, 0.0, 0.0, 7.0)], at, 0.0, 10.0, [(3, 0, 0)], [{"zero_inv": True}])
    # through the corner of voxel (0, 0, 0): x steps first, so (1, 0, 0) is met; z first reaches (1, 1, 1)
    case("corner", [vox((1, 0, 0)), vox((1, 1, 1))], [(1.0, 1.0, 1.0, 0.0)], at, 0.0, 10.0, [(1, 0, 0)],
         [{"tie_z_first": True}])
    # origin on the face x = 0.5 going -x: voxel 1 spans [0, -0) and is passed; the hit is (-1, 0, 0) at 0.5
    case("face_origin", [vox((1, 0, 0)), vox((-1, 0, 0))], [(-1.0, 0.0, 0.0, 0.0)], (0, 0, 0, 0.5, 0.25, 0.25),
         0.0, 10.0, [(-1, 0, 0)], [{"exit_ge": True}])
    # negative coordinates: floor(-0.5) = -1 holds the origin and is occupied
    case("negative", [vox((-1, 0, 0)), vox((2, 0, 0))], [(1.0, 0.0, 0.0, 0.0)], (0, 0, 0, -0.25, 0.25, 0.25),
         0.0, 10.0, [(-1, 0, 0)], [{"trunc": True}])
    # origin inside an occupied voxel: the hit at t = 0 ...
    case("inside", [vox((0, 0, 0)), vox((2, 0, 0))], [(1.0, 0.0, 0.0, 0.0)], at, 0.0, 10.0, [(0, 0, 0)],
         [{"no_normal_exit": True}])
    # ... and with min_range 0.5 beyond its exit at 0.25: (2, 0, 0) at its entry 0.75
    case("inside_beyond", [vox((0, 0, 0)), vox((2, 0, 0))], [(1.0, 0.0, 0.0, 0.0)], at, 0.5, 10.0, [(2, 0, 0)],
         [{"min_ignored": True}])
    # the surfel's plane crosses the ray at 1.4167, beyond the voxel's exit 1.25: clamped to 1.25
    case("surfel_clamp", [vox((2, 0, 0), (-0.6, -0.8, 0.0, 0.0), (1.4, 0.45, 0.25))], [(1.0, 0.0, 0.0, 0.0)], at,
         0.0, 10.0, [(2, 0, 0)], [{"no_clamp": True}])
    # no normal: the entry face, 0.75
    case("no_normal", [vox((2, 0, 0))], [(1.0, 0.0, 0.0, 0.0)], at, 0.0, 10.0, [(2, 0, 0)],
         [{"no_normal_exit": True}])
    # the normal is perpendicular to the ray: den = 0, the entry face
    case("den_zero", [vox((2, 0, 0), (0.0, 1.0, 0.0, 0.0), (1.25, 0.4, 0.25))], [(1.0, 0.0, 0.0, 0.0)], at, 0.0,
         10.0, [(2, 0, 0)], [{"den_zero_divide": True}])
    # the surfel's range is 2.0 exactly: a hit at max_range 2.0 ...
    wall = [vox((4, 0, 0), (-1.0, 0.0, 0.0, 0.0), (2.25, 0.25, 0.25))]
    case("max_exact", wall, [(1.0, 0.0, 0.0, 0.0)], at, 0.0, 2.0, [(4, 0, 0)], [{"max_ge": True}])
    # ... and none at the float below it, though the voxel is entered at 1.75
    case("max_ulp", wall, [(1.0, 0.0, 0.0, 0.0)], at, 0.0, float(np.nextafter(np.float32(2.0), np.float32(0.0))),
         [None], [{"no_t_max": True}])
    # through the corner (-4, -4, -4) of three bricks (voxel -8 starts a brick: -8 + 2^20 is a multiple of 8)
    case("brick_negative", [vox((-8, -9, -9)), vox((-8, -8, -8))], [(1.0, 1.0, 1.0, 0.0)],
         (0, 0, 0, -4.25, -4.25, -4.25), 0.0, 10.0, [(-8, -9, -9)], [{"tie_z_first": True}])
    # the last voxel of a row (2^20 - 1) and beyond: nothing, though the next row's first voxel is occupied
    e = HALF * LEAF
    case("key_range", [vox((-HALF, 1, 0), no, (-e + 0.25, 0.75, 0.25))], [(1.0, 0.0, 0.0, 0.0)],
         (0, 0, 0, e - 0.75, 0.25, 0.25), 0.0, 5.0, [None], [{"wrap": True}])
    # zero and non-finite rays have no hit; a tiny ray is a direction like any other
    case("zero_nonfinite", [vox((2, 0, 0))],
         [(0.0, 0.0, 0.0, 1.0), (np.nan, 1.0, 0.0, 0.0), (np.inf, 0.0, 0.0, 0.0), (1e-30, 0.0, 0.0, 5.0)], at, 0.0,
         10.0, [None, None, None, (2, 0, 0)], [{"zero_eps": True}])
    out = {}
    for k, (c, nrm, r, tw, mn, mx, expect, var) in cases.items():
        out[k] = (np.array(c, np.float32).reshape(-1, 4), np.array(nrm, np.float32).reshape(-1, 4),
                  np.array(r, np.float32).reshape(-1, 4), np.array(tw, np.float32), np.float32(mn), np.float32(mx),
                  expect, var)
    return out


def voxel_index(target, ijk):
    """Position of voxel (i, j, k) in the target, -1 for None."""
    if ijk is None:
        return -1
    return int(lookup(target, np.array([ijk], np.int64))[0])
