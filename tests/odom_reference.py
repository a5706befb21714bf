"""Plain reference of the scan-to-scan correspondence search (BasicLaserOdometry.cpp:246-302 corner, :364-435 surface),
for the tests.

For every query (this sweep's sharp points, then its flat points): transformToStart, the closest point of the last
corner / surface cloud by brute force (fp32 distances ((dx*dx + dy*dy) + dz*dz), every operation rounded, as the
kernel computes them under -fmad=false; the d^2 < 25 gate), then the reference's two serial scan loops from that
closest point.  The loops are restated over index ranges: the forward loop visits j = i1 + 1 .. while j < (the
CURRENT sharp / flat count, an upstream quirk the kernel keeps) and int(intensity) <= scan + 2.5, the backward loop
j = i1 - 1 .. 0 while int(intensity) >= scan - 2.5; the strict `<` updates from 25 keep the first visited of equal
distances, which is the first minimum of the concatenated visiting order.  Nothing here assumes a ring-ordered cloud.

At zero twist transformToStart is exact (s * 0 = 0, sin 0 = 0, cos 1 = 1), so every exact comparison runs there.
"""
from __future__ import annotations

import numpy as np

F = np.float32
GATE = F(25.0)


def ring_ids(cloud):
    """int(intensity): truncation toward zero (C++ float -> int)."""
    return np.trunc(np.asarray(cloud, F)[:, 3]).astype(np.int64)


def sq_dist(cloud, q):
    """fp32 squared distances of every cloud point to q: ((dx*dx + dy*dy) + dz*dz), each operation rounded."""
    p = np.asarray(cloud, F)
    q = np.asarray(q, F)
    dx, dy, dz = p[:, 0] - q[0], p[:, 1] - q[1], p[:, 2] - q[2]
    return (dx * dx + dy * dy) + dz * dz


def transform_to_start(pts, twist6, scan_period=0.1):
    """transformToStart (:40-53) in the kernel's operation order (odometry_lm.cuh: transform_to_start); sin / cos of
    the per-point angles in double, rounded once.  Exact (the identity on xyz) at zero twist."""
    p = np.asarray(pts, F).reshape(-1, 4)
    t = np.asarray(twist6, F).reshape(6)
    inv_sp = F(1.0) / F(scan_period)
    s = inv_sp * (p[:, 3] - np.trunc(p[:, 3]).astype(F))
    x = p[:, 0] - s * t[3]
    y = p[:, 1] - s * t[4]
    z = p[:, 2] - s * t[5]

    def sc(a):
        a = a.astype(np.float64)
        return np.sin(a).astype(F), np.cos(a).astype(F)

    sx, cx = sc(-s * t[0])
    sy, cy = sc(-s * t[1])
    sz, cz = sc(-s * t[2])
    x1 = cz * x - sz * y
    y1 = sz * x + cz * y
    y2 = cx * y1 - sx * z
    z2 = sx * y1 + cx * z
    x3 = cy * x1 + sy * z2
    z3 = cy * z2 - sy * x1
    return np.stack([x3, y2, z3], axis=1).astype(F)


def nearest(d):
    """Closest point from fp32 distances d -> (index, every index tied with it); (-1, []) when d^2 < 25 fails."""
    if d.shape[0] == 0:
        return -1, np.zeros(0, np.int64)
    m = d.min()
    if not m < GATE:
        return -1, np.zeros(0, np.int64)
    ties = np.flatnonzero(d == m)
    return int(ties[0]), ties


def _first_min(d, idx):
    """The serial `if (d < best) { best = d; i = j; }` from best = 25 over candidates in visiting order."""
    ok = d < GATE
    if not ok.any():
        return -1
    d = np.where(ok, d, np.inf)
    return int(idx[int(np.argmin(d))])


def scan_ranges(rings, i1, n_cur):
    """Indices the two serial loops visit from closest point i1: (forward, ascending; backward, descending)."""
    scan = int(rings[i1])
    fend = max(i1 + 1, min(int(n_cur), rings.shape[0]))
    fwd = np.arange(i1 + 1, fend)
    stop = np.flatnonzero(rings[fwd] > scan + 2.5)
    if stop.size:
        fwd = fwd[:stop[0]]
    bwd = np.arange(i1 - 1, -1, -1)
    stop = np.flatnonzero(rings[bwd] < scan - 2.5)
    if stop.size:
        bwd = bwd[:stop[0]]
    return fwd, bwd


def scans_from(last, d, i1, n_cur, corner, rings=None):
    """The two scan loops of one query from a given closest index i1 (d: its fp32 distances to every last point) ->
    (i2, i3); corners have no third point (-1)."""
    if i1 < 0:
        return -1, -1
    rings = ring_ids(last) if rings is None else rings
    scan = int(rings[i1])
    fwd, bwd = scan_ranges(rings, i1, n_cur)
    rf, rb = rings[fwd], rings[bwd]
    if corner:
        cand = np.concatenate([fwd[rf > scan], bwd[rb < scan]])
        return _first_min(d[cand], cand), -1
    c2 = np.concatenate([fwd[rf <= scan], bwd[rb >= scan]])
    c3 = np.concatenate([fwd[rf > scan], bwd[rb < scan]])
    return _first_min(d[c2], c2), _first_min(d[c3], c3)


def scan_margin(last, d, i1, n_cur, corner, which, rings=None):
    """Best and second-best fp32 distance among the candidates of the second (which = 1) or third (which = 2) point."""
    rings = ring_ids(last) if rings is None else rings
    scan = int(rings[i1])
    fwd, bwd = scan_ranges(rings, i1, n_cur)
    idx = np.concatenate([fwd, bwd])
    if corner:
        keep = np.concatenate([rings[fwd] > scan, rings[bwd] < scan])
    elif which == 1:
        keep = np.concatenate([rings[fwd] <= scan, rings[bwd] >= scan])
    else:
        keep = np.concatenate([rings[fwd] > scan, rings[bwd] < scan])
    dd = np.sort(d[idx[keep]])
    dd = dd[dd < GATE]
    return (dd[0] if dd.size else np.inf), (dd[1] if dd.size > 1 else np.inf)


def ulps_apart(a, b):
    """Distance in fp32 ulps of two non-negative finite floats."""
    ia = np.asarray(a, F).view(np.int32).astype(np.int64)
    ib = np.asarray(b, F).view(np.int32).astype(np.int64)
    return np.abs(ia - ib)


class Search:
    """The correspondence search of one iteration (iteration 0, 5, 10, ...) over fixed last clouds."""

    def __init__(self, last_corner, last_surf):
        self.last = (np.ascontiguousarray(last_corner, F).reshape(-1, 4), np.ascontiguousarray(last_surf, F).reshape(-1, 4))
        self.rings = tuple(ring_ids(c) for c in self.last)

    def run(self, sharp, flat, twist6=None):
        """-> dict: ind (n x 3, sharp queries first), ties (per query: indices tied with the closest point), xyz (the
        queries at the start of the sweep), ns (sharp count), n_cur (the forward bounds: sharp and flat counts)."""
        sharp = np.asarray(sharp, F).reshape(-1, 4)
        flat = np.asarray(flat, F).reshape(-1, 4)
        q = np.concatenate([sharp, flat])
        xyz = q[:, :3].copy() if twist6 is None else transform_to_start(q, twist6)
        ns, n = sharp.shape[0], q.shape[0]
        out = {"ind": np.full((n, 3), -1, np.int32), "ties": [None] * n, "xyz": xyz, "ns": ns,
               "n_cur": (ns, flat.shape[0])}
        for kind, lo, hi in ((0, 0, ns), (1, ns, n)):
            last, rings = self.last[kind], self.rings[kind]
            for c0 in range(lo, hi, 32):  # fp32 distance rows of 32 queries at a time
                D = self._dist_rows(last, xyz[c0:min(hi, c0 + 32)])
                for r, d in enumerate(D):
                    k = c0 + r
                    i1, ties = nearest(d)
                    out["ind"][k] = (i1, *scans_from(last, d, i1, out["n_cur"][kind], kind == 0, rings))
                    out["ties"][k] = ties
        return out

    @staticmethod
    def _dist_rows(last, xyz):
        """fp32 squared distances (rows: queries), the operation order of sq_dist."""
        p = last[None, :, :3]
        t = xyz[:, None, :]
        dx, dy, dz = p[..., 0] - t[..., 0], p[..., 1] - t[..., 1], p[..., 2] - t[..., 2]
        return (dx * dx + dy * dy) + dz * dz

    def check(self, res, got, what="", allow_near_ties=0):
        """Compare a GPU index array (n x 3) with run()'s result: i1 equal or an exact fp32 tie with the reference's,
        i2 / i3 equal to the scans from the GPU's own i1.  allow_near_ties: number of queries that may still differ
        where the reference's best and second-best fp32 distances of the differing point are within 4 ulp (non-zero
        twist: per-point sin / cos are not bit-identical).  Returns the number of tie-resolved i1 differences."""
        got = np.asarray(got).reshape(-1, 3)
        ref = res["ind"]
        assert got.shape == ref.shape, (got.shape, ref.shape)
        ns = res["ns"]
        tie_i1 = 0
        bad = []
        for k in np.flatnonzero((got != ref).any(axis=1)):
            corner = k < ns
            last = self.last[0 if corner else 1]
            rings = self.rings[0 if corner else 1]
            n_cur = res["n_cur"][0 if corner else 1]
            d = sq_dist(last, res["xyz"][k])
            g1 = int(got[k, 0])
            if g1 != ref[k, 0]:
                if g1 >= 0 and g1 in set(res["ties"][k].tolist()):
                    tie_i1 += 1
                    exp = scans_from(last, d, g1, n_cur, corner, rings)
                    if (int(got[k, 1]), int(got[k, 2])) == exp:
                        continue
                bad.append((k, "i1", got[k].tolist(), ref[k].tolist(), self._margin_i1(d)))
                continue
            for which in (1, 2):
                if got[k, which] != ref[k, which]:
                    bad.append((k, f"i{which + 1}", got[k].tolist(), ref[k].tolist(),
                                scan_margin(last, d, g1, n_cur, corner, which, rings)))
                    break
        if allow_near_ties:
            near = [b for b in bad if ulps_apart(*b[4]) <= 4]
            assert len(near) == len(bad), f"{what}: differences without a near tie: {[b for b in bad if b not in near][:5]}"
            assert len(bad) <= allow_near_ties, f"{what}: {len(bad)} near-tie differences (at most {allow_near_ties}): {bad[:5]}"
        else:
            assert not bad, f"{what}: {len(bad)} queries differ without an exact tie, e.g. {bad[:5]}"
        return tie_i1

    @staticmethod
    def _margin_i1(d):
        dd = np.sort(d[d < GATE])
        return (dd[0] if dd.size else np.inf), (dd[1] if dd.size > 1 else np.inf)


# ------------------------------------------------------------------------------------------------ test clouds
def last_and_current(drv, lidar, sweep0, scene, yaw_rate):
    """Two consecutive sweeps through the checker's registration: last clouds (less sharp / less flat of sweep0 with
    intensity truncated, as transformToEnd leaves them) and this sweep's sharp / flat."""
    import math

    from loam_velodyne_b200 import synth
    s = drv.scanreg()
    p0, r0 = synth.make_sweep(scene, lidar, sweep0, yaw_rate=math.radians(yaw_rate))
    p1, r1 = synth.make_sweep(scene, lidar, sweep0 + 1, yaw_rate=math.radians(yaw_rate))
    s.process(p0, r0)
    lc, ls = s.cloud("less_sharp").copy(), s.cloud("less_flat").copy()
    lc[:, 3] = np.trunc(lc[:, 3])
    ls[:, 3] = np.trunc(ls[:, 3])
    s.process(p1, r1)
    return lc, ls, s.cloud("sharp").copy(), s.cloud("flat").copy()


def fallback_variants(last_corner, last_surf, seed=3):
    """Last clouds the ring-range fast path must hand over to the serial scan (name -> (corner, surface)):
    rings permuted as blocks, single points moved out of ring order, ring ids remapped to 250..255, rings with gaps in
    their ids, negative intensities."""
    rng = np.random.RandomState(seed)
    out = {}

    def by_ring(c):
        r = ring_ids(c)
        return [c[r == k] for k in np.unique(r)]

    def permuted(c):
        blocks = by_ring(c)
        order = rng.permutation(len(blocks))
        return np.concatenate([blocks[i] for i in order])
    out["rings_permuted"] = (permuted(last_corner), permuted(last_surf))

    def moved(c, n_moves=12):
        c = c.copy()
        for _ in range(n_moves):
            i = rng.randint(0, c.shape[0])
            j = rng.randint(0, c.shape[0])
            row = c[i].copy()
            c = np.delete(c, i, axis=0)
            c = np.insert(c, j, row, axis=0)
        return c
    out["points_moved"] = (moved(last_corner), moved(last_surf))

    def remapped(c):
        c = c.copy()
        r = ring_ids(c)
        c[:, 3] = (250 + r % 6).astype(F)  # keeps the points in place, ring ids 250..255 (not ordered)
        return c

    def remapped_sorted(c):
        c = remapped(c)
        return c[np.argsort(ring_ids(c), kind="stable")]
    out["rings_250_255"] = (remapped(last_corner), remapped(last_surf))
    out["rings_250_255_sorted"] = (remapped_sorted(last_corner), remapped_sorted(last_surf))

    def gaps(c):
        c = c.copy()
        r = ring_ids(c)
        c[:, 3] = (3 * r + 1).astype(F)  # ring-ordered, every second and third id missing
        return c
    out["ring_gaps"] = (gaps(last_corner), gaps(last_surf))

    def negative(c):
        c = c.copy()
        k = rng.choice(c.shape[0], max(1, c.shape[0] // 50), replace=False)
        c[k, 3] = -c[k, 3] - F(0.5)
        return c
    out["negative_intensity"] = (negative(last_corner), negative(last_surf))
    return out


# ------------------------------------------------------------------------------------------------ hand-made edge cases
PAD = np.array([1000.0, 1000.0, 1000.0, 0.0], F)  # a query without any point within 5 m (i1 = -1)


def below_gate():
    """An fp32 offset (a, b, c) whose squared length ((a*a + b*b) + c*c) is the largest float below 25."""
    target = np.nextafter(GATE, F(0))
    b = F(4.0)
    for _ in range(64):
        b = np.nextafter(b, F(0))
        for m in range(0, 4096):
            c = F(m) * F(2.0 ** -12)
            if (F(9.0) + b * b) + c * c == target:
                return np.array([3.0, b, c], F)
    raise AssertionError("no offset found")


def _cloud(spec):
    """spec: (ring, xyz) in cloud order -> n x 4 cloud with intensity = ring."""
    return np.array([(*xyz, float(r)) for r, xyz in spec], F).reshape(-1, 4)


def _fill(ring, k, n):
    """n filler points of a ring, about 4 m from the origin (inside the gate, farther than every crafted candidate)."""
    return [(ring, (0.0, 4.0, 0.01 * (k + i))) for i in range(n)]


def _queries(q, n):
    """Query q first, padded with far queries to n (the forward scans are bound by the query count)."""
    out = np.tile(PAD, (max(n, 1), 1))
    out[0, :3] = q
    out[0, 3] = F(0.5)
    return out[:n]


def _tie(k):
    """The k-th sign variant of (0.3, 0.4, 0.5): equal fp32 squared distance from the origin."""
    sx, sy = (1, -1, 1, -1)[k % 4], (1, 1, -1, -1)[k % 4]
    return (0.3 * sx, 0.4 * sy, 0.5)


I1 = (0.1, 0.0, 0.0)


def edge_cases():
    """name -> (last corner, last surface, sharp, flat): small ring-ordered clouds, queried from the origin at zero
    twist.  The same cloud serves as corner and surface cloud, so each case exercises both kinds of scan."""
    cases = {}

    def add(name, spec, q=(0.0, 0.0, 0.0), n_sharp=None, n_flat=None):
        c = _cloud(spec)
        n = c.shape[0]
        sharp = _queries(q, n if n_sharp is None else n_sharp)
        flat = _queries(q, n if n_flat is None else n_flat)
        cases[name] = (c, c.copy(), sharp, flat)

    g = below_gate()
    # closest point exactly at d^2 = 25 (rejected) / one ulp below (accepted)
    add("gate_closest_at_25", [(0, (0.0, 6.0, 0.0)), (1, (3.0, 4.0, 0.0)), (2, (0.0, 0.0, 6.0))])
    add("gate_closest_below_25", [(0, (0.0, 6.0, 0.0)), (1, tuple(g)), (2, (0.0, 0.0, 6.0))])
    # scan candidates at d^2 = 25 (never taken) and one ulp below (taken): rings 0 / 2 for the corner scans, ring 1
    # forward / backward for the surface's second point
    add("gate_scans", [(0, (3.0, 4.0, 0.0)), (0, (0.0, 6.0, 0.0)), (1, (-3.0, 4.0, 0.0)), (1, I1), (1, (4.0, 3.0, 0.0)),
                       (1, (0.0, 0.0, 5.0)), (2, tuple(-g)), (2, (0.0, -6.0, 0.0))])
    # closest point first / last in the cloud
    line = [(k // 10, (0.5 * k, 0.0, 0.0)) for k in range(50)]
    add("closest_first", line, q=(-0.01, 0.0, 0.0))
    add("closest_last", line, q=(24.51, 0.0, 0.0))
    add("closest_last_backward_only", line, q=(24.51, 0.0, 0.0), n_sharp=3, n_flat=3)
    # the current feature count is below the closest index: the forward scans are empty
    add("count_below_closest", line, q=(12.02, 0.0, 0.0), n_sharp=5, n_flat=5)
    # equidistant candidates: the first visited wins (forward before backward, nearer before farther); the ties sit
    # in different lanes of the warp scans, the one the warp reduction would prefer without the order key is never
    # the first visited
    add("ties_forward_vs_backward", _fill(0, 0, 3) + _fill(1, 3, 1) + [(1, _tie(0)), (1, _tie(2)), (2, I1)] + _fill(2, 4, 5)
        + [(2, _tie(1)), (3, _tie(3))] + _fill(3, 9, 2) + [(3, _tie(1))] + _fill(4, 11, 1))
    add("ties_two_forward", _fill(1, 0, 2) + [(2, I1)] + _fill(3, 2, 7) + [(3, _tie(0))] + _fill(3, 9, 24)
        + [(3, _tie(1))] + _fill(3, 33, 1) + _fill(4, 34, 1))
    add("ties_two_forward_surface", _fill(1, 0, 2) + [(2, I1)] + _fill(2, 2, 7) + [(2, _tie(0))] + _fill(2, 9, 24)
        + [(2, _tie(1))] + _fill(3, 33, 7) + [(3, _tie(2))] + _fill(3, 40, 24) + [(3, _tie(3))] + _fill(4, 64, 1))
    add("ties_two_backward", _fill(0, 0, 1) + [(1, _tie(0))] + _fill(1, 1, 23) + [(1, _tie(1))] + _fill(1, 24, 8)
        + [(2, I1)] + _fill(3, 32, 1) + _fill(4, 33, 1))
    add("ties_two_backward_surface", _fill(0, 0, 1) + [(1, _tie(2))] + _fill(1, 1, 23) + [(1, _tie(3))] + _fill(2, 24, 1)
        + [(2, _tie(0))] + _fill(2, 25, 23) + [(2, _tie(1))] + _fill(2, 48, 8) + [(2, I1)] + _fill(3, 56, 1))
    # the best candidate two rings away (scan + 2 forward, scan - 2 backward): the last rings the scans may visit
    add("reach_two_rings_forward", [(0, (0.3, 0.4, 0.6))] + _fill(0, 0, 1) + _fill(1, 1, 1) + [(2, I1)] + _fill(3, 2, 1)
        + [(4, _tie(1)), (5, _tie(2))] + _fill(5, 3, 1))
    add("reach_two_rings_backward", [(0, _tie(0))] + _fill(1, 0, 2) + [(2, I1)] + _fill(3, 2, 2) + _fill(5, 4, 1)
        + [(5, _tie(1))])
    # empty sharp / empty flat arrays
    c, _, sharp, flat = cases["closest_first"]
    cases["empty_sharp"] = (c, c.copy(), np.zeros((0, 4), F), flat)
    cases["empty_flat"] = (c, c.copy(), sharp, np.zeros((0, 4), F))
    return cases
