"""numpy restatement of the place descriptor and the place match (csrc/densemap.cuh: dense_place_cell,
dense_place_match_kernel; include/loam_b200.h "Place recognition and global relocalisation").

Descriptor, fp64 without FMA (numpy rounds every elementwise operation on its own), per point:
  * skipped when r = sqrt(x*x + z*z) == 0 or r >= max_radius (a non-finite coordinate fails one of these tests or
    the value test);
  * ring = min(floor(r / w), rings - 1), w = max_radius / rings in double;
  * sector = the number of boundaries k in [1, sectors) with past(k): h_p > h_k, or h_p == h_k and
    x * cos(k D) - z * sin(k D) >= 0, D = (2 pi) / sectors, cos / sin of the C library (math.cos / math.sin);
  * value v = (float)(y + height_offset), kept when 0 < v <= FLT_MAX; a cell holds the largest value, 0 when none.
The restatement counts every boundary; the device bisects (past() holds on a prefix of the boundaries).
Distance per candidate and shift s: columns j ascending against candidate column (j + s) mod sectors, qq / dd / dot as
fp64 sums in ascending ring, skip a column with qq == 0 or dd == 0, sim = dot / (sqrt(qq) * sqrt(dd)),
dist = 1 - sum / counted (+inf when none); the best shift is the first smallest.
"""
import math

import numpy as np

F = np.float32
FLT_MAX = float(np.finfo(np.float32).max)


class Params:
    def __init__(self, rings=20, sectors=60, max_radius=80.0, height_offset=2.0, min_range=0.0, max_range=100.0):
        self.rings, self.sectors = int(rings), int(sectors)
        self.max_radius, self.height_offset = float(F(max_radius)), float(F(height_offset))
        self.min_range, self.max_range = float(F(min_range)), float(F(max_range))

    def api(self):
        from loam_velodyne_b200 import api
        return api.PlaceParams(self.rings, self.sectors, F(self.max_radius), F(self.height_offset),
                               F(self.min_range), F(self.max_range))


def step(sectors):
    return (2.0 * math.pi) / sectors


def boundaries(sectors):
    """(cos, sin) of k D for k in [0, sectors), in double from the C library; the boundary at pi (2k == sectors) is
    (-1, 0) exactly."""
    d = step(sectors)
    th = [k * d for k in range(sectors)]
    c, s = np.array([math.cos(t) for t in th]), np.array([math.sin(t) for t in th])
    if sectors % 2 == 0:
        c[sectors // 2], s[sectors // 2] = -1.0, 0.0
    return c, s


def sectors_of(x, z, sectors, edge_gt=False):
    """Sector of each (x, z) by the boundary rule (edge_gt: a deliberately wrong strict test)."""
    c, s = boundaries(sectors)
    hp = np.where((x > 0.0) | ((x == 0.0) & (z > 0.0)), 0, 1)
    count = np.zeros(x.shape, np.int64)
    for k in range(1, sectors):
        hk = 1 if 2 * k >= sectors else 0
        cr = x * c[k] - z * s[k]
        past = (hp > hk) | ((hp == hk) & ((cr > 0.0) if edge_gt else (cr >= 0.0)))
        count += past
    return count


def sectors_atan2(x, z, sectors):
    """Plain binning of atan2(x, z) in [0, 2 pi) (agrees with the rule away from wedge edges)."""
    a = np.mod(np.arctan2(x, z), 2.0 * math.pi)
    return np.minimum(np.floor(a / step(sectors)).astype(np.int64), sectors - 1)


def descriptor(pts, prm, edge_gt=False, ring_ceil=False, r_gt=False, keep_zero_r=False, nan_as_zero=False,
               signed_max=False, last_wins=False, atan2=False):
    """-> float32 (rings, sectors).  The keyword arguments are deliberately wrong variants: a strict boundary test,
    ceil(r / w) - 1 rings, r > max_radius as the only radius cut, r == 0 kept, NaN read as 0, the max over every
    value (an empty cell 0), the last point of a cell wins; atan2: plain azimuth binning."""
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
    if nan_as_zero:
        p = np.where(np.isnan(p), F(0), p)
    x, y, z = (p[:, a].astype(np.float64) for a in range(3))
    with np.errstate(invalid="ignore", over="ignore"):
        r = np.sqrt(x * x + z * z)
        ok = (r <= prm.max_radius) if r_gt else (r < prm.max_radius)
        if not keep_zero_r:
            ok &= r != 0.0
        v = (y + prm.height_offset).astype(np.float32)
        if not signed_max:
            ok &= (v > 0) & (v <= FLT_MAX)
        else:
            ok &= np.isfinite(v)
    x, z, r, v = x[ok], z[ok], r[ok], v[ok]
    w = prm.max_radius / prm.rings
    q = r / w
    ring = (np.ceil(q) - 1.0) if ring_ceil else np.floor(q)
    ring = np.clip(ring, 0, prm.rings - 1).astype(np.int64)
    sec = sectors_atan2(x, z, prm.sectors) if atan2 else sectors_of(x, z, prm.sectors, edge_gt)
    cell = ring * prm.sectors + sec
    if signed_max:
        d = np.full(prm.rings * prm.sectors, -np.inf, np.float32)
        np.maximum.at(d, cell, v)
        d[np.isneginf(d)] = 0.0
    elif last_wins:
        d = np.zeros(prm.rings * prm.sectors, np.float32)
        d[cell] = v
    else:
        d = np.zeros(prm.rings * prm.sectors, np.float32)
        np.maximum.at(d, cell, v)
    return d.reshape(prm.rings, prm.sectors)


def distances(q, d, no_skip=False, shift_sign=False):
    """Distance of query q against candidate d (both (rings, sectors)) at every shift -> float64[sectors].
    no_skip: empty columns count as sim 0; shift_sign: column j against (j - s)."""
    q = np.asarray(q, np.float32).astype(np.float64)
    d = np.asarray(d, np.float32).astype(np.float64)
    R, S = q.shape
    qq = np.zeros(S)
    dd = np.zeros(S)
    for r in range(R):
        qq = qq + q[r] * q[r]
        dd = dd + d[r] * d[r]
    qn, dn = np.sqrt(qq), np.sqrt(dd)
    j = np.arange(S)[None, :]
    s = np.arange(S)[:, None]
    jj = (j - s) % S if shift_sign else (j + s) % S  # (shift, column)
    dot = np.zeros((S, S))
    for r in range(R):
        dot = dot + q[r][None, :] * d[r][jj]
    valid = (qn[None, :] != 0.0) & (dn[jj] != 0.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        sim = dot / (qn[None, :] * dn[jj])
    total = np.zeros(S)
    cnt = np.zeros(S, np.int64)
    for c in range(S):
        if no_skip:
            total = total + np.where(valid[:, c], sim[:, c], 0.0)
            cnt = cnt + 1
        else:
            total = np.where(valid[:, c], total + sim[:, c], total)
            cnt = cnt + valid[:, c]
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(cnt > 0, 1.0 - total / np.maximum(cnt, 1), np.inf)


def best_shift(dist, tie_last=False):
    """(dist, s) of the smallest distance, ties to the smaller s (tie_last: a deliberately wrong larger s)."""
    if tie_last:
        s = len(dist) - 1 - int(np.argmin(dist[::-1]))
    else:
        s = int(np.argmin(dist))
    return float(dist[s]), s


def query(q, db, **variant):
    """Best (dist, shift) of every candidate of db (k, rings, sectors) -> (float64[k], int[k])."""
    tie_last = variant.pop("tie_last", False)
    out = [best_shift(distances(q, d, **variant), tie_last) for d in db]
    return np.array([o[0] for o in out]), np.array([o[1] for o in out], np.int64)


def top_m(dist, m, index_desc=False):
    """Candidates by dist ascending, then index ascending (index_desc: a wrong descending tie), never +inf."""
    idx = np.nonzero(np.isfinite(dist))[0]
    key = -idx if index_desc else idx
    order = idx[np.lexsort((key, dist[idx]))]
    return order[:m]


def yaw_of(s, sectors):
    a = s if 2 * s <= sectors else s - sectors
    return float(np.float32(a * step(sectors)))


def rendered_points(rays, rng):
    """The simulated cloud of a database entry: (float)((double)range_i * u_i) over the rays with a hit, u = p / |p|
    of the cast (rot = 0, so d = u)."""
    p = np.ascontiguousarray(rays, np.float32).reshape(-1, 4)
    x, y, z = (p[:, a].astype(np.float64) for a in range(3))
    ln = np.sqrt((x * x + y * y) + z * z)
    hit = np.isfinite(rng)
    t = rng[hit].astype(np.float32).astype(np.float64)
    u = np.stack([x[hit] / ln[hit], y[hit] / ln[hit], z[hit] / ln[hit]], axis=1)
    out = np.zeros((t.size, 4), np.float32)
    out[:, :3] = (t[:, None] * u).astype(np.float32)
    return out
