"""numpy restatement of carve mode, the ray-walk visibility pass of the whole-run voxel map (csrc/densemap.cuh:
DenseWalk, dense_carve_kernel; include/loam_b200.h "loam_b200_dense_carving").

Per observed cloud, seen from the pose's float position o (taken as double), every point p is one ray; fp64 without
FMA, each operation rounded on its own, in the kernel's order:
  * e = p - o per axis, r = sqrt((ex*ex + ey*ey) + ez*ez), d = e / r; a non-finite p or r == 0 casts nothing, and
    so does every point when the origin's voxel floor(o_a / L) lies outside [-2^20, 2^20);
  * the walk of the ray cast (raycast_reference.cast): start voxel floor(o_a / L), L = (double)leaf; t_next_a =
    ((double)k * L - o_a) * (1.0 / d_a), k = v_a + 1 when d_a > 0, v_a when d_a < 0, +inf when d_a == 0; per voxel
    t_exit = min t_next (ties x, y, z); one step along that axis, only its t_next recomputed from the new index;
  * T = min(r - margin, max_range); the walk ends at the first voxel with t_exit > T (not carved); every voxel
    visited before it that is stored (before this cloud's insertion; indices outside [-2^20, 2^20) never are) is
    carved by the ray;
  * K = the voxels of the cloud's own points (dense_reference.voxel_keys: floorf(c * (1.0f / leaf)));
  * every stored voxel carved by at least one ray and not in K gets one miss, saturating at 65535.
Vectorised over rays, one loop iteration per step; stored voxels are looked up with np.searchsorted on the sorted keys
(the restatement has no bricks: the GPU's occupancy index must not change a bit).
"""
import numpy as np

import dense_reference as dr
import raycast_reference as rr
import visibility_reference as vr

HALF = rr.HALF
MAX_STEPS = rr.MAX_STEPS
SAT = vr.SAT
# recommended parameters (DESIGN.md "Carve mode"), chosen from the margin sweep of tests/test_carve_reference.py
MARGIN, MAX_RANGE = 2.0, 100.0


def lookup(keys, v, wrap=False):
    """Position of the voxels v (M x 3 int64) among the sorted keys, -1 when not stored.  wrap: a deliberately wrong
    variant whose key arithmetic carries an index outside the key range into the next row."""
    u = v + HALF
    if wrap:
        valid = (u >= 0).all(axis=1)
        key = (u[:, 2] << 42) + (u[:, 1] << 21) + u[:, 0]
    else:
        valid = ((v >= -HALF) & (v < HALF)).all(axis=1)
        key = (u[:, 2] << 42) | (u[:, 1] << 21) | u[:, 0]
    m = keys.size
    if m == 0:
        return np.full(v.shape[0], -1, np.int64)
    k = np.where(valid, key, 0).astype(np.uint64)
    pos = np.minimum(np.searchsorted(keys, k), m - 1)
    return np.where(valid & (keys[pos] == k), pos, -1)


def carve_walk(keys, leaf, pts, origin, margin, max_range, max_steps=MAX_STEPS, tie_z_first=False, trunc=False,
               zero_inv=False, exit_lt=False, t_float=False, no_max=False, skip_origin=False, near_as_r=False,
               wrap=False, inf_walks=False):
    """Every carved visit -> (ray index, position among `keys`, t_exit), in walk order per ray.  The keyword arguments
    after max_steps are deliberately wrong variants of the sensitivity tests: ties to z first, a truncated start voxel,
    the t_next formula on an axis with d == 0, t_exit < T, T rounded to float32, no max_range, the origin's voxel never
    carved, T = r when r <= margin, wrapping keys, an infinite point walking to max_range along its sign."""
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
    o = np.array([float(np.float32(x)) for x in origin])
    none = (np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0))
    if p.shape[0] == 0 or keys.size == 0:
        return none
    L = float(np.float32(leaf))
    x, y, z = (p[:, a].astype(np.float64) for a in range(3))
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        ex, ey, ez = x - o[0], y - o[1], z - o[2]
        r = np.sqrt((ex * ex + ey * ey) + ez * ez)
        ok = np.isfinite(p[:, :3]).all(axis=1) & (r > 0.0)
        d = np.stack([ex / r, ey / r, ez / r], axis=1)
        T = np.minimum(r - float(margin), float(max_range)) if not no_max else r - float(margin)
    if inf_walks:
        inf = np.isinf(p[:, :3]).any(axis=1) & ~np.isnan(p[:, :3]).any(axis=1)
        d[inf] = np.where(np.isinf(p[inf, :3]), np.sign(p[inf, :3]), 0.0)
        T[inf] = float(max_range)
        ok |= inf
    if near_as_r:
        T = np.where(r <= float(margin), r, T)
    if t_float:
        T = T.astype(np.float32).astype(np.float64)
    rows = np.nonzero(ok)[0]
    d, T = d[rows], T[rows]
    m = rows.size
    so = np.floor(o / L)
    if not ((so >= -HALF) & (so < HALF)).all():  # an origin outside the key range casts nothing
        return none
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
    first = np.ones(m, bool)
    act = np.arange(m)
    out_r, out_j, out_t = [], [], []
    for _ in range(max_steps):
        if act.size == 0:
            break
        x, y, z = tn[act, 0], tn[act, 1], tn[act, 2]
        if tie_z_first:
            ax = np.where((z <= y) & (z <= x), 2, np.where(y <= x, 1, 0))
        else:
            ax = np.where((x <= y) & (x <= z), 0, np.where(y <= z, 1, 2))
        tx = tn[act, ax]
        go = (tx < T[act]) if exit_lt else (tx <= T[act])
        act, ax, tx = act[go], ax[go], tx[go]
        if act.size == 0:
            break
        j = lookup(keys, v[act], wrap)
        h = j >= 0
        if skip_origin:
            h &= ~first[act]
        if h.any():
            out_r.append(rows[act[h]])
            out_j.append(j[h])
            out_t.append(tx[h])
        first[act] = False
        fwd = d[act, ax] > 0.0
        v[act, ax] += np.where(fwd, 1, -1)
        k = np.where(fwd, v[act, ax] + 1, v[act, ax])
        with np.errstate(invalid="ignore"):
            tn[act, ax] = (k.astype(np.float64) * L - o[ax]) * inv[act, ax]
    if not out_r:
        return none
    return np.concatenate(out_r), np.concatenate(out_j), np.concatenate(out_t)


def ray_ranges(pts, origin):
    """r per point, as the walk computes it (NaN for a non-finite point)."""
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
    o = np.array([float(np.float32(x)) for x in origin])
    with np.errstate(invalid="ignore", over="ignore"):
        e = p[:, :3].astype(np.float64) - o
        return np.sqrt((e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2])


def miss_mask(keys, leaf, pts, carved, no_k=False):
    """Stored voxels (positions among keys) that get a miss: carved by some ray, not in K.  no_k: the deliberately
    wrong variant without the K exclusion."""
    hit = np.zeros(keys.size, bool)
    hit[carved] = True
    if not no_k and keys.size:
        k = np.unique(dr.voxel_keys(pts, leaf))
        k = k[k != dr.EMPTY]
        pos = np.minimum(np.searchsorted(keys, k), keys.size - 1)
        hit[pos[keys[pos] == k]] = False
    return hit


class CarveMapRef(vr.VisibilityMapRef):
    """VisibilityMapRef whose pass is carve mode (max_range > 0) instead of the range image."""

    def __init__(self, leaf, max_voxels=2**31 - 1, margin=MARGIN, max_range=MAX_RANGE, **variants):
        super().__init__(leaf, max_voxels)
        self.set_carving(margin, max_range)
        self.variants = variants

    def set_carving(self, margin, max_range):
        self.c_margin, self.c_max = float(margin), float(max_range)

    def carved(self, pts, twist6):
        """Positions (among self.keys) of the stored voxels the cloud's rays carve, with repetitions."""
        v = {k: x for k, x in self.variants.items() if k not in ("no_k", "per_ray", "no_sat")}  # the walk's variants
        t6 = np.asarray(twist6, np.float32)
        return carve_walk(self.keys, self.leaf, pts, t6[3:6], self.c_margin, self.c_max, **v)[1]

    def observe(self, pts, twist6):
        if not (self.c_max > 0.0):
            return super().observe(pts, twist6)
        if self.keys.size == 0 or np.asarray(pts).size == 0:
            return
        j = self.carved(pts, twist6)
        miss = miss_mask(self.keys, self.leaf, pts, j, self.variants.get("no_k", False)).astype(np.int64)
        if self.variants.get("per_ray"):
            miss = np.bincount(j, minlength=self.keys.size) * miss
        m = self.misses + miss
        self.misses = m if self.variants.get("no_sat") else np.minimum(m, SAT)


def slab(keys, leaf, pts, origin):
    """Per finite ray with r > 0: for every stored voxel, its slab entry max(t_near, 0) and exit t_far along d = e / r
    (computed independently of the walk) -> (rows, entry R x M, exit R x M, T-free r R)."""
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
    o = np.array([float(np.float32(x)) for x in origin])
    L = float(np.float32(leaf))
    e = p[:, :3].astype(np.float64) - o
    r = np.sqrt((e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2])
    rows = np.nonzero(np.isfinite(p[:, :3]).all(axis=1) & (r > 0.0))[0]
    d = e[rows] / r[rows, None]
    vox = dr.key_voxel(keys)
    lo_b, hi_b = vox * L, (vox + 1) * L
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / d
        t1 = (lo_b[None] - o) * inv[:, None, :]
        t2 = (hi_b[None] - o) * inv[:, None, :]
    par = (d == 0.0)[:, None, :]
    inside = ((lo_b <= o) & (o < hi_b))[None]
    t1 = np.where(par, np.where(inside, -np.inf, np.inf), t1)
    t2 = np.where(par, np.where(inside, np.inf, -np.inf), t2)
    tn = np.minimum(t1, t2).max(axis=2)
    tf = np.maximum(t1, t2).min(axis=2)
    return rows, np.maximum(tn, 0.0), tf, r[rows]


# ---- hand-made cases
LEAF = rr.LEAF  # 0.5: every coordinate below is exact in fp32; 1 / leaf is exact


def _c(i, j, k):
    return ((i + 0.5) * LEAF, (j + 0.5) * LEAF, (k + 0.5) * LEAF, 1.0)


def edge_cases():
    """{name: (stored points M x 4, observed cloud N x 4, origin, margin, max_range, expected misses per stored voxel in
    key order, variants, repeat)}: each variant (keyword arguments of CarveMapRef) is a deliberately wrong restatement
    that changes the misses on that case; repeat = how many times the cloud is observed."""
    at = (0.25, 0.25, 0.25)  # inside voxel (0, 0, 0)
    cases = {}

    def case(name, stored, seen, origin, margin, mx, expect, variants, repeat=1):
        cases[name] = (np.array(stored, np.float32).reshape(-1, 4), np.array(seen, np.float32).reshape(-1, 4),
                       origin, margin, mx, expect, variants, repeat)

    # d_y = d_z = 0: t_next is +inf on those axes (the formula there walks -y and -z instead)
    case("axis_parallel", [_c(2, 0, 0)], [(4.25, 0.25, 0.25, 1.0)], at, 0.5, 50.0, [1], [{"zero_inv": True}])
    # through the corner of voxel (0, 0, 0): x steps first, so (1, 0, 0) is crossed; z first crosses (0, 0, 1)
    case("corner", [_c(1, 0, 0), _c(0, 0, 1)], [(2.75, 2.75, 2.75, 1.0)], at, 0.5, 50.0, [1, 0],
         [{"tie_z_first": True}])
    # the origin inside a stored voxel: carved like any other
    case("origin_inside", [_c(0, 0, 0)], [(3.25, 0.25, 0.25, 1.0)], at, 0.5, 50.0, [1], [{"skip_origin": True}])
    # r = 1.75, margin 1: T = 0.75 = the exit of voxel (1, 0, 0): carved ...
    case("exit_exact", [_c(1, 0, 0)], [(2.0, 0.25, 0.25, 1.0)], at, 1.0, 50.0, [1], [{"exit_lt": True}])
    # ... and one double more margin: T one ulp below 0.75, not carved (T rounded to float would carve)
    case("exit_ulp", [_c(1, 0, 0)], [(2.0, 0.25, 0.25, 1.0)], at, float(np.nextafter(1.0, 2.0)), 50.0, [0],
         [{"t_float": True}])
    # max_range 2: voxel (4, 0, 0) exits at 2.25 > 2, voxel (3, 0, 0) at 1.75 is carved
    case("max_range", [_c(3, 0, 0), _c(4, 0, 0)], [(10.25, 0.25, 0.25, 1.0)], at, 0.5, 2.0, [1, 0],
         [{"no_max": True}])
    # r <= margin (the point in voxel (-1, 0, 0)): T < 0, nothing carved, not even the origin's voxel
    case("near", [_c(0, 0, 0)], [(-0.05, 0.25, 0.25, 1.0)], at, 0.5, 50.0, [0], [{"near_as_r": True}])
    # (1, 0, 0) is crossed by one ray and holds another's return: in K, no miss; (2, 0, 0) is carved: a miss
    case("crossed_in_k", [_c(1, 0, 0), _c(2, 0, 0)], [(3.25, 0.25, 0.25, 1.0), (0.75, 0.3, 0.3, 1.0)], at, 0.5, 50.0,
         [0, 1], [{"no_k": True}])
    # many rays through one voxel: one miss
    fan = [(4.25, 0.25 + 0.01 * i, 0.25 + 0.013 * i, 1.0) for i in range(8)]
    case("many_rays", [_c(1, 0, 0)], fan, at, 0.5, 50.0, [1], [{"per_ray": True}])
    # saturation: observed 3 times from a count of 65533
    case("saturation", [_c(1, 0, 0)], [(4.25, 0.25, 0.25, 1.0)], at, 0.5, 50.0, [SAT], [{"no_sat": True}], repeat=3)
    # negative coordinates through the corner of bricks (voxel -8 starts a brick): floor, not trunc, of the origin
    case("brick_negative", [_c(-9, -9, -9), _c(-8, -8, -8)], [(-1.75, -1.75, -1.75, 1.0)], (-4.25, -4.25, -4.25),
         0.2, 50.0, [1, 1], [{"trunc": True}])
    # the last voxel of a row (2^20 - 1) and beyond: the next row's first voxel is never carved
    e = HALF * LEAF
    case("key_range", [(-e + 0.25, 0.75, 0.25, 1.0), (e - 0.25, 0.25, 0.25, 1.0)], [(e + 2.25, 0.25, 0.25, 1.0)],
         (e - 0.75, 0.25, 0.25), 0.5, 50.0, [1, 0], [{"wrap": True}])
    # zero and non-finite points cast nothing
    case("zero_nonfinite", [_c(1, 0, 0), _c(-2, 0, 0)],
         [(0.25, 0.25, 0.25, 1.0), (np.nan, 1.0, 0.0, 1.0), (np.inf, 0.25, 0.25, 1.0), (-np.inf, 0.25, 0.25, 1.0)],
         at, 0.5, 50.0, [0, 0], [{"inf_walks": True}])
    return cases


def run_case(name, **variants):
    stored, seen, origin, margin, mx, _, _, repeat = edge_cases()[name]
    ref = CarveMapRef(LEAF, margin=margin, max_range=mx, **variants)
    ref.insert(stored)
    if name == "saturation":
        ref.misses[:] = SAT - 2
    tw = np.array([0.0, 0.0, 0.0, *origin], np.float32)
    for _ in range(repeat):
        ref.observe(seen, tw)
    return ref


def margin_sweep(run, leaf, margins, max_range=MAX_RANGE, ratio=1.0, settle=6):
    """Trail removed / static kept of carve mode at every margin over one moving-box run (vr.moving_box_run) -> {margin:
    (removed, kept)}.  The stored set does not depend on the misses, so each sweep is walked once at the smallest
    margin and the carved visits of the others are the prefixes with t_exit <= min(r - margin, max_range)."""
    trail, static = vr.trail_and_static(run, leaf, settle)
    base = vr.VisibilityMapRef(leaf)
    m0 = min(margins)
    misses = {m: None for m in margins}
    for pts, twist, _ in run:
        keys = base.keys
        if keys.size:
            ray, j, t = carve_walk(keys, leaf, pts, np.asarray(twist, np.float32)[3:6], m0, max_range)
            r = ray_ranges(pts, np.asarray(twist, np.float32)[3:6])[ray]
            for m in margins:
                sel = t <= np.minimum(r - m, max_range)
                miss = miss_mask(keys, leaf, pts, j[sel]).astype(np.int64)
                misses[m] = np.minimum(misses[m] + miss, SAT)
        base.insert(pts)
        for m in margins:  # re-align the counters with the new key set
            old = misses[m]
            new = np.zeros(base.keys.size, np.int64)
            if old is not None and keys.size:
                new[np.searchsorted(base.keys, keys)] = old
            misses[m] = new
    out = {}
    for m in margins:
        base.misses = misses[m]
        out[m] = vr.removal_rates(base, trail, static, ratio)
    return out
