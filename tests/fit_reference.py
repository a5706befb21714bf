"""Plain restatement of the four per-correspondence fits of the two Gauss-Newton loops, for the tests.

* fp32, the reference arithmetic: ``map_corner_fit`` / ``map_surf_fit`` (BasicLaserMapping.cpp:671-816) and
  ``odom_corner_fit`` / ``odom_surf_fit`` (BasicLaserOdometry.cpp:319-356, 400-476) in numpy float32 scalar operations,
  in the source's order.  The 3x3 eigen-decomposition and the 5x3 least-squares solve come from the checker
  (``Driver.eig_sym`` / ``Driver.lsq53``, the oracle's Eigen restatement); they are not restated here.
* float64, an independent answer: the same formulas on the same fp32 inputs with numpy.linalg.eigh / lstsq, with the
  distance of every decision from its threshold.
* ``cases(seed, drv)`` / ``odom_cases(seed)``: a catalogue of isolated neighbourhoods aimed at the degenerate branches
  of csrc/linalg.cuh and of the residuals.

Every fit returns ``(selected, coeff[4])``; coeff is zero where the reference leaves the coefficient unwritten.
"""
from __future__ import annotations

import itertools

import numpy as np

F = np.float32
D = np.float64
FLT_MIN = np.finfo(np.float32).tiny
EPS32 = float(np.finfo(np.float32).eps)
ZERO4 = np.zeros(4, np.float32)


def _f3(p):
    p = np.asarray(p, np.float32).reshape(-1)
    return F(p[0]), F(p[1]), F(p[2])


# ---------------------------------------------------------------------------------------------- fp32 restatement
def line_residual(q, p1, p2):
    """BasicLaserMapping.cpp:712-730 / BasicLaserOdometry.cpp:319-337 -> (la, lb, lc, ld2), all float32."""
    x0, y0, z0 = _f3(q)
    x1, y1, z1 = _f3(p1)
    x2, y2, z2 = _f3(p2)
    with np.errstate(all="ignore"):
        m11 = (x0 - x1) * (y0 - y2) - (x0 - x2) * (y0 - y1)
        m12 = (x0 - x1) * (z0 - z2) - (x0 - x2) * (z0 - z1)
        m13 = (y0 - y1) * (z0 - z2) - (y0 - y2) * (z0 - z1)
        a012 = np.sqrt(m11 * m11 + m12 * m12 + m13 * m13)
        l12 = np.sqrt((x1 - x2) * (x1 - x2) + (y1 - y2) * (y1 - y2) + (z1 - z2) * (z1 - z2))
        la = ((y1 - y2) * m11 + (z1 - z2) * m12) / a012 / l12
        lb = -((x1 - x2) * m11 - (z1 - z2) * m13) / a012 / l12
        lc = -((x1 - x2) * m12 + (y1 - y2) * m13) / a012 / l12
        ld2 = a012 / l12
    return la, lb, lc, ld2


def corner_covariance(nn):
    """Centroid (sequential sums, / 5.0f) and the 3x3 covariance / 5 (lower triangle, upper zero) in fp32."""
    nn = np.asarray(nn, np.float32)[:5, :3]
    vx = vy = vz = F(0)
    for j in range(5):
        vx = vx + nn[j, 0]
        vy = vy + nn[j, 1]
        vz = vz + nn[j, 2]
    vx, vy, vz = vx / F(5), vy / F(5), vz / F(5)
    m = np.zeros((3, 3), np.float32)
    for j in range(5):
        ax, ay, az = nn[j, 0] - vx, nn[j, 1] - vy, nn[j, 2] - vz
        m[0, 0] += ax * ax
        m[1, 0] += ax * ay
        m[2, 0] += ax * az
        m[1, 1] += ay * ay
        m[2, 1] += ay * az
        m[2, 2] += az * az
    return (vx, vy, vz), m / F(5)


def map_corner_fit(drv, nn, q):
    (vx, vy, vz), m = corner_covariance(nn)
    ev, V = drv.eig_sym(m)
    if not ev[2] > F(3) * ev[1]:
        return False, ZERO4.copy()
    # end points vc +- 0.1 * v: the 0.1 literal is a double (BasicLaserMapping.cpp:705-710)
    e1 = [F(D(v) + 0.1 * D(V[i, 2])) for i, v in enumerate((vx, vy, vz))]
    e2 = [F(D(v) - 0.1 * D(V[i, 2])) for i, v in enumerate((vx, vy, vz))]
    la, lb, lc, ld2 = line_residual(q, e1, e2)
    with np.errstate(all="ignore"):
        s = F(1) - F(0.9) * np.abs(ld2)
        coeff = np.array([s * la, s * lb, s * lc, s * ld2], np.float32)
    return bool(D(s) > 0.1), coeff


def map_surf_fit(drv, nn, q):
    nn = np.asarray(nn, np.float32)[:5, :3]
    x = drv.lsq53(nn)
    with np.errstate(all="ignore"):
        pa, pb, pc, pd = F(x[0]), F(x[1]), F(x[2]), F(1)
        ps = np.sqrt(pa * pa + pb * pb + pc * pc)
        pa, pb, pc, pd = pa / ps, pb / ps, pc / ps, pd / ps
        for j in range(5):
            if D(np.abs(pa * nn[j, 0] + pb * nn[j, 1] + pc * nn[j, 2] + pd)) > 0.2:
                return False, ZERO4.copy()
        sx, sy, sz = _f3(q)
        pd2 = pa * sx + pb * sy + pc * sz + pd
        s = F(1) - F(0.9) * np.abs(pd2) / np.sqrt(np.sqrt(sx * sx + sy * sy + sz * sz))
        coeff = np.array([s * pa, s * pb, s * pc, s * pd2], np.float32)
    return bool(D(s) > 0.1), coeff


def odom_corner_fit(t1, t2, q, it):
    la, lb, lc, ld2 = line_residual(q, t1, t2)
    with np.errstate(all="ignore"):
        s = F(1)
        if it >= 5:
            s = F(1) - F(1.8) * np.abs(ld2)
        coeff = np.array([s * la, s * lb, s * lc, s * ld2], np.float32)
    return bool(D(s) > 0.1 and ld2 != 0), coeff


def odom_surf_fit(t1, t2, t3, q, it):
    x1, y1, z1 = _f3(t1)
    x2, y2, z2 = _f3(t2)
    x3, y3, z3 = _f3(t3)
    sx, sy, sz = _f3(q)
    with np.errstate(all="ignore"):
        pa = (y2 - y1) * (z3 - z1) - (y3 - y1) * (z2 - z1)
        pb = (z2 - z1) * (x3 - x1) - (z3 - z1) * (x2 - x1)
        pc = (x2 - x1) * (y3 - y1) - (x3 - x1) * (y2 - y1)
        pd = -(pa * x1 + pb * y1 + pc * z1)
        ps = np.sqrt(pa * pa + pb * pb + pc * pc)
        pa, pb, pc, pd = pa / ps, pb / ps, pc / ps, pd / ps
        pd2 = pa * sx + pb * sy + pc * sz + pd
        s = F(1)
        if it >= 5:
            s = F(1) - F(1.8) * np.abs(pd2) / np.sqrt(np.sqrt(sx * sx + sy * sy + sz * sz))
        coeff = np.array([s * pa, s * pb, s * pc, s * pd2], np.float32)
    return bool(D(s) > 0.1 and pd2 != 0), coeff


# ---------------------------------------------------------------------------------------------- branch probes (fp32)
def eigen_v1norm2(nn):
    """v1norm2 of sym_eigen<3>'s closed-form tridiagonalisation: (m[2] / scale)^2 in fp32 (<= FLT_MIN: shortcut)."""
    _, m = corner_covariance(nn)
    low = np.abs(np.tril(m))
    scale = F(low.max()) if low.max() != 0 else F(1)
    m2 = m[2, 0] / scale
    return m2, m2 * m2


def colpiv_branches(nn):
    """The control flow of colpiv_qr_solve<5, 3> on A = nn (fp32, the same operations as csrc/linalg.cuh): returns
    dict(nonzero, recomputed = number of norm down-dates that fell back to recomputation, pivot_tie = a pivot
    choice among exactly equal column norms) and the solution, which the tests pin to the checker's lsq53."""
    A = np.array(np.asarray(nn, np.float32)[:5, :3], np.float32, copy=True)
    b = np.full(5, F(-1), np.float32)
    R, C = 5, 3
    nDir = np.array([np.sqrt(np.float32(sum_sq(A[:, k]))) for k in range(C)], np.float32)
    nUpd = nDir.copy()
    perm = list(range(C))
    maxNorm = F(0)
    for k in range(C):
        if nUpd[k] > maxNorm:
            maxNorm = nUpd[k]
    thr0 = maxNorm * F(EPS32)
    helper = thr0 * thr0 / F(R)
    dthr = np.sqrt(F(EPS32))
    nonzero, recomputed, tie = C, 0, False
    h = np.zeros(C, np.float32)
    with np.errstate(all="ignore"):
        for k in range(C):
            big, bigNorm = k, nUpd[k]
            for j in range(k + 1, C):
                if nUpd[j] > bigNorm:
                    bigNorm, big = nUpd[j], j
            tie = tie or any(nUpd[j] == bigNorm and j != big for j in range(k, C))
            if nonzero == C and bigNorm * bigNorm < helper * F(R - k):
                nonzero = k
            if big != k:
                A[:, [k, big]] = A[:, [big, k]]
                nUpd[[k, big]] = nUpd[[big, k]]
                nDir[[k, big]] = nDir[[big, k]]
                perm[k], perm[big] = perm[big], perm[k]
            tail = F(0)
            for i in range(k + 1, R):
                tail = tail + A[i, k] * A[i, k]
            c0 = A[k, k]
            if R - k == 1 or tail <= FLT_MIN:
                tau, beta = F(0), c0
                A[k + 1:, k] = 0
            else:
                beta = np.sqrt(c0 * c0 + tail)
                if c0 >= 0:
                    beta = -beta
                den = c0 - beta
                for i in range(k + 1, R):
                    A[i, k] = A[i, k] / den
                tau = (beta - c0) / beta
            h[k] = tau
            A[k, k] = beta
            if tau != 0:
                for j in range(k + 1, C):
                    t = F(0)
                    for i in range(k + 1, R):
                        t = t + A[i, k] * A[i, j]
                    t = t + A[k, j]
                    A[k, j] = A[k, j] - tau * t
                    for i in range(k + 1, R):
                        A[i, j] = A[i, j] - tau * A[i, k] * t
            for j in range(k + 1, C):
                if nUpd[j] != 0:
                    t = np.abs(A[k, j]) / nUpd[j]
                    t = (F(1) + t) * (F(1) - t)
                    t = F(0) if t < 0 else t
                    ratio = nUpd[j] / nDir[j]
                    if t * (ratio * ratio) <= dthr:
                        s = F(0)
                        for i in range(k + 1, R):
                            s = s + A[i, j] * A[i, j]
                        nDir[j] = np.sqrt(s)
                        nUpd[j] = nDir[j]
                        recomputed += 1
                    else:
                        nUpd[j] = nUpd[j] * np.sqrt(t)
        x = np.zeros(C, np.float32)
        if nonzero > 0:
            for k in range(nonzero):
                if h[k] != 0:
                    t = F(0)
                    for i in range(k + 1, R):
                        t = t + A[i, k] * b[i]
                    t = t + b[k]
                    b[k] = b[k] - h[k] * t
                    for i in range(k + 1, R):
                        b[i] = b[i] - h[k] * A[i, k] * t
            for i in range(nonzero - 1, -1, -1):
                v = b[i]
                for l in range(i + 1, nonzero):
                    v = v - A[i, l] * b[l]
                b[i] = v / A[i, i]
            for i in range(nonzero):
                x[perm[i]] = b[i]
    return {"nonzero": nonzero, "recomputed": recomputed, "pivot_tie": tie}, x


def sum_sq(col):
    s = F(0)
    for v in np.asarray(col, np.float32):
        s = s + v * v
    return s


# ---------------------------------------------------------------------------------------------- float64 answer
def _line64(q, p1, p2):
    x0, y0, z0 = q
    x1, y1, z1 = p1
    x2, y2, z2 = p2
    m11 = (x0 - x1) * (y0 - y2) - (x0 - x2) * (y0 - y1)
    m12 = (x0 - x1) * (z0 - z2) - (x0 - x2) * (z0 - z1)
    m13 = (y0 - y1) * (z0 - z2) - (y0 - y2) * (z0 - z1)
    a012 = np.sqrt(m11 * m11 + m12 * m12 + m13 * m13)
    l12 = np.sqrt((x1 - x2) ** 2 + (y1 - y2) ** 2 + (z1 - z2) ** 2)
    with np.errstate(all="ignore"):
        return (np.array([((y1 - y2) * m11 + (z1 - z2) * m12) / a012 / l12,
                          -((x1 - x2) * m11 - (z1 - z2) * m13) / a012 / l12,
                          -((x1 - x2) * m12 + (y1 - y2) * m13) / a012 / l12]), a012 / l12)


def map_corner_fit64(nn, q):
    """-> (selected, coeff, margins, cond).  margins: (ev2 - 3 ev1) / ev2 and s - 0.1; cond bounds the error of the
    line direction and of the centroid subtraction: (1 + |centroid| / spread) * ev2 / (ev2 - ev1)."""
    p = np.asarray(nn, np.float32)[:5, :3].astype(D)
    q = np.asarray(q, np.float32)[:3].astype(D)
    c = p.mean(axis=0)
    a = p - c
    w, V = np.linalg.eigh(a.T @ a / 5.0)
    spread = np.sqrt(max(w[2], 0.0))
    gap = w[2] - w[1]
    cond = (1.0 + np.abs(c).max() / spread) * w[2] / gap if gap > 0 and spread > 0 else np.inf
    ev_margin = (w[2] - 3.0 * w[1]) / w[2] if w[2] > 0 else -np.inf
    if not w[2] > 3.0 * w[1]:
        return False, np.zeros(4), {"ev": ev_margin}, cond
    l, ld2 = _line64(q, c + 0.1 * V[:, 2], c - 0.1 * V[:, 2])
    s = 1.0 - 0.9 * abs(ld2)
    return bool(s > 0.1), np.append(s * l, s * ld2), {"ev": ev_margin, "s": s - 0.1}, cond


def map_surf_fit64(nn, q):
    """-> (selected, coeff, margins, cond).  margins: 0.2 - largest plane residual and s - 0.1 (absolute); cond is
    the 2-norm condition number of the 5 x 3 system (inf when rank deficient)."""
    A = np.asarray(nn, np.float32)[:5, :3].astype(D)
    q = np.asarray(q, np.float32)[:3].astype(D)
    sv = np.linalg.svd(A, compute_uv=False)
    cond = sv[0] / sv[2] if sv[2] > 0 else np.inf
    x = np.linalg.lstsq(A, -np.ones(5), rcond=None)[0]
    ps = np.linalg.norm(x)
    with np.errstate(all="ignore"):
        n, pd = x / ps, 1.0 / ps
    res = np.abs(A @ n + pd).max()
    if res > 0.2:
        return False, np.zeros(4), {"valid": 0.2 - res}, cond
    pd2 = n @ q + pd
    s = 1.0 - 0.9 * abs(pd2) / np.sqrt(np.linalg.norm(q))
    return bool(s > 0.1), np.append(s * n, s * pd2), {"valid": 0.2 - res, "s": s - 0.1}, cond


def near_threshold(margins, rel=1e-6):
    return any(abs(v) <= rel for v in margins.values())


# ---------------------------------------------------------------------------------------------- NaN-aware bits
def same_bits(a, b):
    """Per row: every float equal bit for bit, or both NaN (the NaN payload is not compared)."""
    a = np.ascontiguousarray(a, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    eq = (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))
    return eq.reshape(eq.shape[0], -1).all(axis=1) if eq.ndim > 1 else eq


# ---------------------------------------------------------------------------------------------- the catalogue
# Every neighbourhood is 5 map points around one query, isolated: lattice sites are 5 m apart (so the 5-NN within 1 m
# of the query is exactly the cluster), the rest sit in their own batch.  Distinct points have distinct fp32 distances
# from the query, so the neighbour order is fixed.  Coordinates are in the map frame.
LATTICE_X = [10.0 + 5.0 * i for i in range(19)]          # x = 10 .. 100
LATTICE_Z = [-100.0 + 5.0 * i for i in range(41)]        # z = -100 .. 100, y = 0: inside the 125 cubes around 0


def sq_dist(p, q):
    """fp32 squared distances in the order of the searches (dx * dx + dy * dy + dz * dz)."""
    p = np.asarray(p, np.float32)[:, :3]
    d = p - np.asarray(q, np.float32)[:3]
    return d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]


def order_neighbours(pts, q):
    """Points sorted by fp32 distance from q; raises unless only identical points share a distance and all are
    within 1 m."""
    pts = np.asarray(pts, np.float32)[:, :3]
    d = sq_dist(pts, q)
    o = np.argsort(d, kind="stable")
    pts, d = pts[o], d[o]
    assert d[-1] < 1.0, f"neighbour at d^2 = {d[-1]}"
    for i in range(4):
        assert d[i] != d[i + 1] or np.array_equal(pts[i], pts[i + 1]), f"distance tie {d[i]}"
    return pts


class Case:
    def __init__(self, name, family, kind, pts, q, target, batch="lattice", ties=False):
        self.name, self.family, self.kind, self.target, self.batch = name, family, kind, target, batch
        self.q = np.asarray(q, np.float32)[:3].copy()
        self.pts = np.asarray(pts, np.float32)[:, :3].copy() if ties else order_neighbours(pts, self.q)

    def __repr__(self):
        return f"Case({self.name})"


def _site(k):
    return np.array([LATTICE_X[k % len(LATTICE_X)], 0.0, LATTICE_Z[k // len(LATTICE_X)]], np.float32)


def _crossing(above, lo, hi):
    """Adjacent floats (a, b) in [lo, hi] (both positive) with above(a) != above(b), by bisection on the bit patterns
    (above(lo) != above(hi) is required)."""
    a, b = int(F(lo).view(np.int32)), int(F(hi).view(np.int32))
    fa = above(np.int32(a).view(np.float32))
    assert fa != above(np.int32(b).view(np.float32)), (lo, hi)
    while b - a > 1:
        m = (a + b) // 2
        if above(np.int32(m).view(np.float32)) == fa:
            a = m
        else:
            b = m
    return np.int32(a).view(np.float32), np.int32(b).view(np.float32)


def _ev_ratio_cases(drv, c):
    """ev2 == 3 ev1 exactly in fp32, and one float either side: points (cx +- 0.5, 0, cz), (cx, +-b, cz), (cx, 0, cz)
    with b stepped float by float around 0.5 / sqrt(3) (y = 0 on the lattice, so b is fine-grained)."""
    found = {}
    # b steps 3 ev1 by ~3 floats at a time, the fifth point's y (e) fills in between; a moves ev2 (3 ev1 cannot
    # round to every float)
    for a, e in itertools.product(range(16), range(100)):
        a = F(0.5) + F(a) / F(1024)
        b0 = F(a / np.sqrt(3.0))
        for db in range(-4, 5):
            b = b0 + F(db) * np.spacing(b0)
            pts = np.array([[c[0] + a, 0, c[2]], [c[0] - a, 0, c[2]], [c[0], b, c[2]], [c[0], -b, c[2]],
                            [c[0], F(e) * F(1e-5), c[2]]], np.float32)
            _, m = corner_covariance(pts)
            ev, _ = drv.eig_sym(m)
            three = F(3) * ev[1]
            for key, hit in (("eq", ev[2] == three), ("above", ev[2] == np.nextafter(three, F(np.inf))),
                             ("below", ev[2] == np.nextafter(three, F(-np.inf)))):
                if hit and key not in found:
                    found[key] = pts
        if len(found) == 3:
            break
    assert len(found) == 3, f"ev2 == 3 ev1 edges not found: {sorted(found)}"
    return found


def _valid_edge_cases(drv, c, q):
    """Largest plane residual equal to 0.2f (> 0.2 in double: invalid) and to the float below (valid): plane
    y = c + 0.5 = 0.05 with the fifth point lifted by about 0.25 m.  The residual's last term (pd) must be small for
    every float near 0.2 to be reachable: with the plane metres from the origin the residual is a difference of
    numbers near pd and moves in steps of 16 floats of 0.2."""
    found = {}
    want = {"at_0.2f": F(0.2), "below_0.2f": np.nextafter(F(0.2), F(0))}

    def make(y5, dx):
        y = c[1] + F(0.5)
        return order_neighbours(np.array([[c[0] + 0.4, y, c[2] + 0.3], [c[0] - 0.4, y, c[2] + 0.2],
                                          [c[0] + 0.1, y, c[2] - 0.4], [c[0] - 0.2, y, c[2] - 0.3],
                                          [c[0] + dx, y5, c[2]]], np.float32), q)  # the order the fit sees

    def res(pts):
        x = drv.lsq53(pts)
        with np.errstate(all="ignore"):
            pa, pb, pc = F(x[0]), F(x[1]), F(x[2])
            ps = np.sqrt(pa * pa + pb * pb + pc * pc)
            pa, pb, pc, pd = pa / ps, pb / ps, pc / ps, F(1) / ps
            return max(np.abs(pa * p[0] + pb * p[1] + pc * p[2] + pd) for p in pts)

    # the fifth point's y by bisection, then float by float; its x in small steps fills in between
    for i in range(400):
        dx = F(i) * F(1e-7)
        lo, _ = _crossing(lambda y: res(make(y, dx)) > F(0.2), c[1] + F(0.6), c[1] + F(0.9))
        for y in (np.nextafter(lo, F(0)), lo, np.nextafter(lo, F(9))):
            r = res(make(y, dx))
            for key, v in want.items():
                if r == v and key not in found:
                    found[key] = make(y, dx)
        if len(found) == 2:
            break
    assert len(found) == 2, f"0.2 residual edges not found: {sorted(found)}"
    return found


def _surf_s_edge_cases(drv):
    """s = 1 - 0.9 |pd2| / |q|^(1/2) on both sides of 0.1 (the two achievable values around it): only reachable
    with the query near the sensor origin.  Plane y = 0.75, query (0.03, y, 0.02), y stepped float by float."""
    pts = np.array([[0.4, 0.75, 0.3], [-0.4, 0.75, 0.35], [0.3, 0.75, -0.4], [-0.35, 0.75, -0.3], [0.05, 0.75, 0.45]],
                   np.float32)
    x = drv.lsq53(pts)
    pa, pb, pc = F(x[0]), F(x[1]), F(x[2])
    ps = np.sqrt(pa * pa + pb * pb + pc * pc)
    pa, pb, pc, pd = pa / ps, pb / ps, pc / ps, F(1) / ps

    def make(y):
        return np.array([0.03, y, 0.02], np.float32)

    def s_of(q):
        pd2 = pa * q[0] + pb * q[1] + pc * q[2] + pd
        return F(1) - F(0.9) * np.abs(pd2) / np.sqrt(np.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]))

    lo, hi = _crossing(lambda y: D(s_of(make(y))) > 0.1, F(0.2), F(0.3))
    above, below = (hi, lo) if D(s_of(make(hi))) > 0.1 else (lo, hi)
    return pts, {"above": (make(above), s_of(make(above))), "below": (make(below), s_of(make(below)))}


def cases(seed, drv):
    """The mapping catalogue: a list of Case.  `drv` is the checker (its eig_sym / lsq53 find the exact edges)."""
    rng = np.random.RandomState(seed)
    out = []
    k = [0]

    def site():
        c = _site(k[0])
        k[0] += 1
        return c

    def add(name, family, kind, pts, q, target, **kw):
        out.append(Case(name, family, kind, pts, q, target, **kw))

    # ---- corner fits
    for i, d in enumerate(((3, -2, 1), (1, 1, 1), (-5, 2, 7))):
        c = site()
        d = np.asarray(d, np.float32) / F(64)
        t = np.array([-6, -2, 1, 3, 5], np.float32)
        add(f"corner_collinear_general_{i}", "collinear_general", "corner", c + t[:, None] * d,
            c + np.array([0.11, 0.2, -0.15], np.float32), "exactly collinear, m[2] != 0")
    for ax in range(3):
        c = site()
        t = np.array([-5, -2, 0.5, 3, 6], np.float32) / F(8)
        pts = np.repeat(c[None], 5, axis=0)
        pts[:, ax] += t
        off = np.array([0.05, 0.3, 0.2], np.float32)
        add(f"corner_collinear_axis{'xyz'[ax]}", "collinear_axis", "corner", pts, c + off,
            "exactly collinear along an axis: m[2] == 0, FLT_MIN shortcut")
    for i, e in enumerate((1e-19, 3e-20)):
        c = np.array([0.0, 0.0, -40.0 - 6.0 * i], np.float32)  # x ~ 0: offsets of 1e-19 are representable
        pts = np.array([[0, -0.6, c[2]], [e, -0.2, c[2] + 0.01], [-e, 0.1, c[2] - 0.02], [2 * e, 0.4, c[2] + 0.03],
                        [0, 0.7, c[2]]], np.float32)
        add(f"corner_m2_subnormal_{i}", "m2_tiny", "corner", pts, np.array([0.1, 0.07, c[2] + 0.2], np.float32),
            "0 < m[2]^2 <= FLT_MIN: shortcut with m[2] != 0", batch="x0")
    c = site()
    add("corner_identical", "identical", "corner", np.repeat((c + F(0.125))[None], 5, axis=0),
        c + np.array([0.1, -0.2, 0.3], np.float32), "5 identical points: zero matrix")
    for i, (a, b) in enumerate(((0.5, 0.5), (0.25, 0.25))):
        c = site()
        pts = c + np.array([[a, 0, 0], [-a, 0, 0], [0, 0, b], [0, 0, -b], [0, 0, 0]], np.float32)
        add(f"corner_planar_tie_{i}", "planar", "corner", pts, c + np.array([0.11, 0.07, 0.05], np.float32),
            "planar, two equal large eigenvalues")
    c = site()
    pts = c + (rng.uniform(-0.5, 0.5, (5, 3)) * np.array([1, 0, 1])).astype(np.float32)
    add("corner_planar_random", "planar", "corner", pts, c + np.array([0.05, 0.1, 0.0], np.float32),
        "planar random")
    for i, pat in enumerate((((0.5, 0, 0), (-0.5, 0, 0), (0, 0.5, 0), (0, -0.5, 0), (0, 0, 0)),
                             ((0, 0.5, 0), (0, -0.5, 0), (0, 0, 0.5), (0, 0, -0.5), (0, 0, 0)),
                             ((0.75, 0, 0), (-0.75, 0, 0), (0, 0.25, 0), (0, 0, 0.25), (0, -0.25, -0.25)),
                             ((0.5, 0.5, 0), (-0.5, -0.5, 0), (0.5, -0.5, 0), (-0.5, 0.5, 0), (0, 0, 0)))):
        c = site()
        add(f"corner_axis_ties_{i}", "axis_ties", "corner", c + np.array(pat, np.float32),
            c + np.array([0.13, 0.06, 0.09], np.float32), "+-axis pattern, eigenvalue ties")
    c = site()
    for key, pts in _ev_ratio_cases(drv, c).items():
        add(f"corner_ev_ratio_{key}", "ev_ratio_edge", "corner", pts, c + np.array([0.02, 0.05, 0.3], np.float32),
            "ev2 == 3 ev1 in fp32 (eq), one float above / below", batch=f"ev_{key}")
    for i in range(3):
        c = site()
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        t = np.array([-2, -1, 0, 1, 2.5])[:, None]
        pts = (c + 1e-4 * (t * d + 0.05 * rng.normal(size=(5, 3)))).astype(np.float32)
        add(f"corner_spread_1e-4_{i}", "tiny_spread", "corner", pts, c + np.array([0.01, 0.2, 0.1], np.float32),
            "1e-4 m spread (coordinates quantised to a few ulp)")
    for i in range(4):
        c = np.array([3000.0 + 5.0 * i, 20.0, 3000.0], np.float32)
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        pts = (c + np.array([-0.6, -0.25, 0.05, 0.3, 0.55])[:, None] * d + 0.02 * rng.normal(size=(5, 3))).astype(np.float32)
        add(f"corner_far_3km_{i}", "far_3km", "corner", pts, c + np.array([0.1, 0.15, -0.1], np.float32),
            "3 km from the origin: centroid subtraction cancels", batch="far")
    for ax in range(3):
        c = site()
        pts = np.repeat(c[None], 5, axis=0)
        pts[:, ax] += np.array([-0.5, -0.25, 0.125, 0.375, 0.625], np.float32)
        q = c.copy()
        q[ax] += F(0.03125)
        add(f"corner_query_on_line_{'xyz'[ax]}", "query_on_line", "corner", pts, q,
            "query on the fitted line: a012 == 0, NaN coefficient, selected", batch="poison")
    for i in range(12):
        c = site()
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        pts = (c + rng.uniform(-0.45, 0.45, (5, 1)) * d + 0.03 * rng.normal(size=(5, 3))).astype(np.float32)
        add(f"corner_random_{i}", "random", "corner", pts, c + (0.15 * rng.normal(size=3)).astype(np.float32).clip(-0.2, 0.2),
            "general line")

    # ---- surface fits
    for ax in range(3):
        c = site()
        off = np.array([[0.3, 0.2, -0.4], [-0.4, 0.3, 0.1], [0.1, -0.45, 0.3], [-0.2, -0.1, -0.3], [0.45, 0.4, 0.4]],
                       np.float32)
        off[:, ax] = F(0.25) if ax == 1 else 0
        add(f"surf_axis_plane_{'xyz'[ax]}", "axis_plane", "surf", c + off, c + np.array([0.05, 0.1, 0.15], np.float32),
            "axis-aligned plane: one constant column")
    c = site()
    pts = c + np.array([[0.3, 0, -0.4], [-0.4, 0, 0.1], [0.1, 0, 0.3], [-0.2, 0, -0.3], [0.45, 0, 0.4]], np.float32)
    add("surf_origin_plane_y0", "origin_plane", "surf", pts, c + np.array([0.05, 0.2, 0.1], np.float32),
        "plane y = 0 through the sensor origin: zero column, rank 2")
    for i, (t0, v0) in enumerate(((1.0, 0.0), (1.0, 0.001))):
        c = site()
        tt = np.array([-0.003, -0.0015, 0.0, 0.002, 0.003]) + t0
        vv = np.array([-0.4, 0.3, -0.1, 0.2, 0.45])
        pts = np.stack([c[0] * tt, vv, c[2] * tt], axis=1).astype(np.float32)
        pts[:, 0] += F(v0)
        add(f"surf_origin_plane_diag_{i}", "origin_plane", "surf", pts, c + np.array([0.1, 0.05, -0.1], np.float32),
            "plane through (or 1e-3 m from) the sensor origin: A x = -1 ill-conditioned")
    c = site()
    pts = c + np.array([[0.3, 0.001, -0.4], [-0.4, 0.001, 0.1], [0.1, 0.001, 0.3], [-0.2, 0.001, -0.3],
                        [0.45, 0.001, 0.4]], np.float32) - np.array([0, c[1], 0], np.float32)
    add("surf_origin_plane_y1mm", "origin_plane", "surf", pts, c + np.array([0.05, 0.2, 0.1], np.float32),
        "plane y = 1e-3 m")
    c = site()
    d = np.array([3, -2, 1], np.float32) / F(32)
    add("surf_collinear", "collinear", "surf", c + np.array([-6, -2, 1, 3, 5], np.float32)[:, None] * d,
        c + np.array([0.1, 0.2, -0.2], np.float32), "5 collinear points: rank 2")
    c = site()
    add("surf_identical", "identical", "surf", np.repeat((c + F(0.125))[None], 5, axis=0),
        c + np.array([0.1, -0.2, 0.3], np.float32), "5 identical points: rank 1")
    add("surf_all_at_origin", "origin_points", "surf", np.zeros((5, 3), np.float32),
        np.array([0.2, 0.1, 0.3], np.float32), "all points at the origin: nonzero == 0, ps = 0, NaN", batch="origin")
    o = np.array([-0.5, -0.25, 0.0, 0.25, 0.5], np.float32)
    for name, c, perm in (("xz", np.array([40.0, 0.0, 40.0], np.float32), (None, [1, 3, 0, 4, 2])),
                          ("xyz", np.array([40.0, 40.0, 40.0], np.float32), ([2, 0, 4, 1, 3], [1, 3, 0, 4, 2]))):
        pts = np.repeat(c[None], 5, axis=0)
        pts[:, 0] += o
        pts[:, 1] += o[perm[0]] if perm[0] is not None else np.array([0.1, -0.3, 0.2, 0.35, -0.15], np.float32)
        pts[:, 2] += o[perm[1]]
        add(f"surf_equal_norms_{name}", "pivot_ties", "surf", pts, c + np.array([0.03, 0.11, 0.07], np.float32),
            "columns with exactly equal norms: pivot ties", batch=f"ties_{name}")
    for i, eps in enumerate((1e-3, 3e-5)):
        c = site()
        c[2] = c[0]
        base = np.array([-0.5, -0.2, 0.1, 0.3, 0.45], np.float32)
        pts = np.stack([c[0] + base, np.array([0.3, -0.4, 0.1, -0.2, 0.4]), c[0] + base + F(eps) * np.array([1, -1, 2, 0, -2])],
                       axis=1).astype(np.float32)
        add(f"surf_near_parallel_{i}", "near_parallel", "surf", pts, c + np.array([0.02, 0.1, -0.05], np.float32),
            "nearly parallel columns: norm down-date recomputed", batch=f"par_{i}")
    c = np.array([0.0, -0.45, 0.0], np.float32)
    q = c + np.array([0.05, 0.55, 0.02], np.float32)
    for key, pts in _valid_edge_cases(drv, c, q).items():
        add(f"surf_valid_{key}", "valid_edge", "surf", pts, q,
            "largest plane residual one float either side of 0.2 (double compare)", batch=f"valid_{key}")
    c = site()
    pts = c + np.array([[0.3, 0.2, 0], [-0.4, 0.3, 0], [0.1, -0.45, 0], [-0.2, -0.1, 0], [0.45, 0.4, 0]], np.float32)
    add("surf_query_on_plane", "query_on_plane", "surf", pts, c + np.array([0.05, 0.1, 0.0], np.float32),
        "query on the plane")
    spts, edges = _surf_s_edge_cases(drv)
    for key, (q, _) in edges.items():
        add(f"surf_s_{key}_0.1", "s_edge", "surf", spts, q, "s one step either side of 0.1 (query near the origin)",
            batch=f"s_{key}")
    for i in range(12):
        c = site()
        n = rng.normal(size=3)
        n /= np.linalg.norm(n)
        u = np.cross(n, [0.3, 0.5, 0.7])
        u /= np.linalg.norm(u)
        v = np.cross(n, u)
        ab = rng.uniform(-0.5, 0.5, (5, 2))
        pts = (c + ab[:, :1] * u + ab[:, 1:] * v + 0.02 * rng.normal(size=(5, 1)) * n).astype(np.float32)
        add(f"surf_random_{i}", "random", "surf", pts, (c + 0.2 * n + 0.05 * rng.normal(size=3)).astype(np.float32),
            "general plane")
    names = [cs.name for cs in out]
    assert len(set(names)) == len(names)
    return out


def ordered_alternatives(pts, q):
    """Every ordering of `pts` consistent with a sort by fp32 distance from q (permutations within exact ties)."""
    pts = np.asarray(pts, np.float32)[:, :3]
    d = sq_dist(pts, q)
    o = np.argsort(d, kind="stable")
    groups = [list(g) for _, g in itertools.groupby(o, key=lambda i: d[i])]
    for combo in itertools.product(*[itertools.permutations(g) for g in groups]):
        yield pts[[i for g in combo for i in g]]


def tie_cases():
    """Clusters with two or three neighbours at exactly the same fp32 distance from the query."""
    out = []
    for i, (pat, q) in enumerate((
            (((0.5, 0, 0), (-0.5, 0, 0), (0, 0.3, 0.1), (0, -0.2, 0.4), (0.1, 0.1, -0.3)), (0, 0, 0)),
            (((0.5, 0, 0), (0, 0.5, 0), (0, 0, 0.5), (-0.3, -0.1, 0), (0.2, -0.2, -0.35)), (0, 0, 0)),
            (((0.25, 0.5, 0), (-0.25, 0.5, 0), (0.25, -0.5, 0), (-0.25, -0.5, 0), (0, 0, 0.4)), (0, 0, 0)))):
        c = np.array([-60.0 - 5.0 * i, 0.0, 60.0], np.float32)
        for kind in ("corner", "surf"):
            out.append(Case(f"{kind}_ties_{i}", "ties", kind, c + np.array(pat, np.float32), c + np.array(q, np.float32),
                            "exactly equidistant neighbours", batch="ties", ties=True))
    return out


# ---------------------------------------------------------------------------------------------- odometry catalogue
class OdomCase:
    """A correspondence in the last clouds: line (t1, t2) or plane (t1, t2, t3) and one query."""

    def __init__(self, name, family, kind, pts, q, target, batch="finite", tie_pair=False):
        self.name, self.family, self.kind, self.target, self.batch = name, family, kind, target, batch
        self.pts = np.asarray(pts, np.float32)[:, :3]
        self.q = np.asarray(q, np.float32)[:3]
        self.tie_pair = tie_pair  # t1 and t2 coincide: the closest point is either of them


def _weight_edges(fit, make, lo, hi):
    """The two adjacent query coordinates in [lo, hi] between which the weight s of iterations >= 5 crosses 0.1."""
    a, b = _crossing(lambda v: D(fit(make(v))) > 0.1, lo, hi)
    above, below = (a, b) if D(fit(make(a))) > 0.1 else (b, a)
    return {"above": make(above), "below": make(below)}


def _odom_line_s(t1, t2, q):
    _, _, _, ld2 = line_residual(q, t1, t2)
    return F(1) - F(1.8) * np.abs(ld2)


def _odom_plane_s(t1, t2, t3, q):
    x1, y1, z1 = _f3(t1)
    x2, y2, z2 = _f3(t2)
    x3, y3, z3 = _f3(t3)
    sx, sy, sz = _f3(q)
    pa = (y2 - y1) * (z3 - z1) - (y3 - y1) * (z2 - z1)
    pb = (z2 - z1) * (x3 - x1) - (z3 - z1) * (x2 - x1)
    pc = (x2 - x1) * (y3 - y1) - (x3 - x1) * (y2 - y1)
    pd = -(pa * x1 + pb * y1 + pc * z1)
    ps = np.sqrt(pa * pa + pb * pb + pc * pc)
    pa, pb, pc, pd = pa / ps, pb / ps, pc / ps, pd / ps
    pd2 = pa * sx + pb * sy + pc * sz + pd
    return F(1) - F(1.8) * np.abs(pd2) / np.sqrt(np.sqrt(sx * sx + sy * sy + sz * sz))


def odom_cases(seed):
    """The odometry catalogue: a list of OdomCase, every one 12 m from the next (the 1-NN radius is 5 m)."""
    rng = np.random.RandomState(seed)
    out = []
    k = [0]

    def site():
        c = np.array([20.0 + 12.0 * (k[0] % 8), 2.0, -40.0 + 12.0 * (k[0] // 8)], np.float32)
        k[0] += 1
        return c

    def add(*a, **kw):
        out.append(OdomCase(*a, **kw))

    c = site()
    p = c + np.array([0.3, -0.2, 0.1], np.float32)
    add("odom_line_coincident", "coincident", "corner", [p, p], c + np.array([0.5, 0.4, 0.2], np.float32),
        "t1 == t2: l12 = 0, inf / NaN coefficient, selected below iteration 5", batch="poison", tie_pair=True)
    c = site()
    d = np.array([0.25, -0.125, 0.5], np.float32)
    add("odom_plane_collinear", "plane_collinear", "surf", [c, c + d, c - d], c + np.array([0.3, 0.2, -0.1], np.float32),
        "three collinear plane points: ps = 0, NaN, selected below iteration 5", batch="poison")
    for ax in range(3):
        c = site()
        e = np.zeros(3, np.float32)
        e[ax] = F(0.5)
        add(f"odom_query_on_line_{'xyz'[ax]}", "query_on_line", "corner", [c, c + e], c + F(0.125) * e,
            "query on the line: ld2 == 0 (not selected), NaN coefficient")
    c = site()
    on = np.array([[0, 0, 0], [0.5, 0.25, 0], [-0.25, 0.5, 0]], np.float32) + c
    add("odom_query_on_plane", "query_on_plane", "surf", on, c + np.array([0.1, 0.2, 0.0], np.float32),
        "query on the plane: pd2 == 0 (not selected)")
    # s = 1 - 1.8 |ld2| and 1 - 1.8 |pd2| / |q|^(1/2) on both sides of 0.1 (the weight of iterations >= 5)
    for key in ("above", "below"):  # each on its own site: the two queries would otherwise share t1, t2
        c = site()
        t1, t2 = c, c + np.array([0.5, 0.0, 0.0], np.float32)
        q = _weight_edges(lambda q: _odom_line_s(t1, t2, q), lambda y: np.array([c[0] + 0.05, y, c[2]], np.float32),
                          c[1] + F(0.4), c[1] + F(0.6))[key]
        add(f"odom_line_weight_{key}", "weight_edge", "corner", [t1, t2], q, "s = 1 - 1.8 |ld2| either side of 0.1")
    for key in ("above", "below"):
        c = site()
        pl = [c, c + np.array([0.5, 0, 0.0], np.float32), c + np.array([0, 0, 0.5], np.float32)]
        norm = float(np.linalg.norm(c)) ** 0.5
        q = _weight_edges(lambda q: _odom_plane_s(*pl, q), lambda y: np.array([c[0] + 0.1, y, c[2] + 0.1], np.float32),
                          c[1] + F(0.3 * norm), c[1] + F(0.7 * norm))[key]
        add(f"odom_plane_weight_{key}", "weight_edge", "surf", pl, q, "s = 1 - 1.8 |pd2| / |q|^(1/2) either side of 0.1")

    def unit():
        d = rng.normal(size=3)
        return d / np.linalg.norm(d)

    for i in range(6):  # t2, t3 1 m from t1, the query within 0.35 m of t1: t1 is the closest point
        c = site()
        add(f"odom_line_random_{i}", "random", "corner", [c, (c + unit()).astype(np.float32)],
            (c + 0.2 * rng.uniform(-1, 1, 3)).astype(np.float32), "general line")
        c = site()
        add(f"odom_plane_random_{i}", "random", "surf",
            [c, (c + unit()).astype(np.float32), (c + unit()).astype(np.float32)],
            (c + 0.2 * rng.uniform(-1, 1, 3)).astype(np.float32), "general plane")
    return out


FAR = np.array([0.0, 900.0, 0.0], np.float32)  # padding queries: no last point within 5 m


def odom_clouds(cs):
    """Last corner / surface clouds and sharp / flat queries for a list of OdomCase.  Ring ids (intensity) are chosen
    so that the reference's scans pick the intended points: a line's t1 on ring 3 and t2 on ring 2 (found by the
    backward scan, ring < scan); a plane's t3 on ring 2, t2 on ring 3 just before t1 (same ring, backward scan).  The
    query arrays are padded past the last clouds' sizes because the forward scans are bounded by the current
    feature counts (BasicLaserOdometry.cpp:262, :378).  Returns (lc, ls, sharp, flat, expected indices per case)."""
    lines = [c for c in cs if c.kind == "corner"]
    planes = [c for c in cs if c.kind == "surf"]
    lc = np.zeros((2 * len(lines), 4), np.float32)
    for i, c in enumerate(lines):
        lc[i, :3], lc[i, 3] = c.pts[1], 2.0
        lc[len(lines) + i, :3], lc[len(lines) + i, 3] = c.pts[0], 3.0
    ls = np.zeros((3 * len(planes), 4), np.float32)
    for i, c in enumerate(planes):
        ls[i, :3], ls[i, 3] = c.pts[2], 2.0
        ls[len(planes) + 2 * i, :3], ls[len(planes) + 2 * i, 3] = c.pts[1], 3.0
        ls[len(planes) + 2 * i + 1, :3], ls[len(planes) + 2 * i + 1, 3] = c.pts[0], 3.0
    exp = {}
    for i, c in enumerate(lines):
        exp[c.name] = (len(lines) + i, i, -1)
    for i, c in enumerate(planes):
        exp[c.name] = (len(planes) + 2 * i + 1, len(planes) + 2 * i, i)

    def queries(group, n_min):
        q = np.zeros((max(len(group), n_min), 4), np.float32)
        q[:, :3] = FAR
        for i, c in enumerate(group):
            q[i, :3] = c.q
        q[:, 3] = 5.0  # integral intensity: relative time 0, transformToStart is the identity
        return q

    return lc, ls, queries(lines, lc.shape[0] + 1), queries(planes, ls.shape[0] + 1), exp
