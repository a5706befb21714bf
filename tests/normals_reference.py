"""numpy restatement of the normals of the whole-run voxel map's export (csrc/densemap.cuh: dense_normals_kernel;
include/loam_b200.h "loam_b200_dense_export_normals").

Input: an exported cloud -- its keys (ascending, as dense_reference / visibility_reference keep them) and fp32
centroids -- plus the radius (1..3) and the viewpoint.  Only the voxels given are neighbours: a voxel the miss-ratio
filter removed is simply not in the input.  Every floating-point operation is the kernel's, in the kernel's order:
  * neighbours of v: the voxels whose index differs by at most `radius` on every axis, v included, visited in ascending
    key order (dz, then dy, then dx ascending); an offset outside [-2^20, 2^20) on an axis does not exist;
  * fp64, each operation rounded on its own: d = (double)c_w - (double)c_v; S1 += d; S2 += d_a * d_b for xx, xy, xz,
    yy, yz, zz; k neighbours; C_ab = (float)((S2_ab - (S1_a * S1_b) / k) / k);
  * eigen-decomposition of C by the checker (Driver.eig_sym: Eigen's SelfAdjointEigenSolver<Matrix3f>, which the
    device's sym_eigen<3> equals bit for bit); normal = eigenvector of the smallest eigenvalue; curvature =
    ev0 / ((ev0 + ev1) + ev2) in fp32, 0 when that sum is 0;
  * flip when ((p_x - c_x) * n_x + (p_y - c_y) * n_y) + (p_z - c_z) * n_z < 0 in double;
  * k < 3: NaN normal and curvature.  (The checker's solver does not report non-convergence, which the kernel maps to
    NaN as well; a 3 x 3 symmetric matrix converges within the iteration cap.)
The sums are vectorised over voxels, one offset at a time in the order above, and never use np.sum (pairwise).
"""
import numpy as np

import dense_reference as dr

HALF = dr.HALF
NAN32 = np.float32(np.nan)  # 0x7fc00000, the kernel's NaN


def offsets(radius):
    """(dx, dy, dz) in visiting order: dz, then dy, then dx, each ascending."""
    r = range(-radius, radius + 1)
    return [(dx, dy, dz) for dz in r for dy in r for dx in r]


def pack(v):
    """(N, 3) int64 voxel indices inside the key range -> uint64 keys."""
    u = (np.asarray(v, np.int64) + HALF).astype(np.uint64)
    return (u[:, 2] << np.uint64(42)) | (u[:, 1] << np.uint64(21)) | u[:, 0]


def neighbour(keys, vox, off):
    """Keys of the voxels at offset `off` from every voxel, and whether that offset stays inside the key range."""
    w = vox + np.asarray(off, np.int64)
    ok = np.all((w >= -HALF) & (w < HALF), axis=1)
    k = np.zeros(vox.shape[0], np.uint64)
    k[ok] = pack(w[ok])
    return k, ok


def sums(keys, cent, radius, neighbour_fn=neighbour):
    """-> S1 (N, 3), S2 (N, 6: xx, xy, xz, yy, yz, zz) in fp64 and k (N,) over each voxel's neighbours.

    An absent neighbour adds +0.0 to every sum.  That is exact: the sums start at +0.0, and in round-to-nearest a sum
    is -0.0 only when both addends are -0.0, so no sum is ever -0.0, and s + (+0.0) == s for every other s (a present
    neighbour can add -0.0 through a product, which leaves the sum as it is for the same reason)."""
    keys = np.asarray(keys, np.uint64)
    c = np.asarray(cent, np.float32).reshape(-1, 4)[:, :3].astype(np.float64)
    n = keys.size
    vox = dr.key_voxel(keys)
    S1 = np.zeros((n, 3), np.float64)
    S2 = np.zeros((n, 6), np.float64)
    k = np.zeros(n, np.int64)
    if n == 0:
        return S1, S2, k
    for off in offsets(radius):
        wk, ok = neighbour_fn(keys, vox, off)
        pos = np.minimum(np.searchsorted(keys, wk), n - 1)
        found = ok & (keys[pos] == wk)
        d = np.where(found[:, None], c[pos] - c, 0.0)
        S1 = S1 + d
        a, b = [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]
        S2 = S2 + d[:, a] * d[:, b]
        k = k + found
    return S1, S2, k


def covariance(S1, S2, k):
    """-> (N, 3, 3) fp32 symmetric covariances (each entry (S2_ab - (S1_a * S1_b) / k) / k rounded once)."""
    kd = np.maximum(k, 1).astype(np.float64)[:, None]
    a, b = [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]
    e = ((S2 - (S1[:, a] * S1[:, b]) / kd) / kd).astype(np.float32)
    C = np.empty((k.size, 3, 3), np.float32)
    for j, (p, q) in enumerate(zip(a, b)):
        C[:, p, q] = e[:, j]
        C[:, q, p] = e[:, j]
    return C


def finish(C, k, cent, viewpoint, drv, min_k=3, flip_le=False):
    """Eigen-decomposition, curvature and orientation -> (N, 4) float32 (nx, ny, nz, curvature).  min_k and flip_le
    exist for the tests that show the edge cases would catch a wrong threshold or a non-strict flip."""
    c = np.asarray(cent, np.float32).reshape(-1, 4)[:, :3].astype(np.float64)
    p = np.asarray(viewpoint, np.float64).reshape(3)
    out = np.full((k.size, 4), NAN32, np.float32)
    for i in np.nonzero(k >= min_k)[0]:
        ev, V = drv.eig_sym(C[i])
        nrm = V[:, 0].astype(np.float32)
        den = (ev[0] + ev[1]) + ev[2]  # float32 scalars: each sum rounds to fp32
        curv = np.float32(0.0) if den == 0 else np.float32(ev[0] / den)
        f = ((p[0] - c[i, 0]) * float(nrm[0]) + (p[1] - c[i, 1]) * float(nrm[1])) + (p[2] - c[i, 2]) * float(nrm[2])
        if f < 0.0 or (flip_le and f == 0.0):
            nrm = -nrm
        out[i, :3] = nrm
        out[i, 3] = curv
    return out


def normals(keys, cent, radius, viewpoint, drv=None, **variant):
    """The exported cloud (ascending keys, N x 4 fp32 centroids) -> (N, 4) float32 (nx, ny, nz, curvature)."""
    if drv is None:
        from oracle import pydriver
        drv = pydriver.best()
    S1, S2, k = sums(keys, cent, radius, variant.pop("neighbour_fn", neighbour))
    return finish(covariance(S1, S2, k), k, cent, viewpoint, drv, **variant)


def normals_loop(keys, cent, radius, viewpoint, drv):
    """The same, one voxel at a time with Python floats (IEEE double, no FMA) and a dict of keys: the plain reading of
    the specification, against which the vectorised version is checked."""
    keys = np.asarray(keys, np.uint64)
    cent = np.asarray(cent, np.float32).reshape(-1, 4)
    where = {int(kk): j for j, kk in enumerate(keys)}
    vox = dr.key_voxel(keys)
    out = np.full((keys.size, 4), NAN32, np.float32)
    for i in range(keys.size):
        cx, cy, cz = (float(cent[i, a]) for a in range(3))
        s1 = [0.0, 0.0, 0.0]
        s2 = [0.0] * 6
        k = 0
        for dx, dy, dz in offsets(radius):
            w = (int(vox[i, 0]) + dx, int(vox[i, 1]) + dy, int(vox[i, 2]) + dz)
            if not all(-HALF <= x < HALF for x in w):
                continue
            j = where.get(((w[2] + HALF) << 42) | ((w[1] + HALF) << 21) | (w[0] + HALF))
            if j is None:
                continue
            d = (float(cent[j, 0]) - cx, float(cent[j, 1]) - cy, float(cent[j, 2]) - cz)
            for a in range(3):
                s1[a] += d[a]
            for m, (a, b) in enumerate(((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))):
                s2[m] += d[a] * d[b]
            k += 1
        if k < 3:
            continue
        C = np.zeros((3, 3), np.float32)
        for m, (a, b) in enumerate(((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))):
            C[a, b] = C[b, a] = np.float32((s2[m] - (s1[a] * s1[b]) / k) / k)
        ev, V = drv.eig_sym(C)
        nrm = V[:, 0].astype(np.float32)
        den = (ev[0] + ev[1]) + ev[2]
        curv = np.float32(0.0) if den == 0 else np.float32(ev[0] / den)
        p = [float(x) for x in viewpoint]
        if ((p[0] - cx) * float(nrm[0]) + (p[1] - cy) * float(nrm[1])) + (p[2] - cz) * float(nrm[2]) < 0.0:
            nrm = -nrm
        out[i, :3] = nrm
        out[i, 3] = curv
    return out


EDGE_LEAF = 0.5  # 1 / leaf is exact, and every coordinate below is a multiple of 1/16, exact in fp32 up to 2^19 m
LAST = HALF - 1  # the last voxel index of an axis; -HALF is the first


def _block(xs, ys, zs, rng, per=3):
    """Points in every voxel of xs x ys x zs (indices), at jittered eighths of the voxel, so centroids differ."""
    pts = []
    for z in zs:
        for y in ys:
            for x in xs:
                f = rng.randint(1, 8, (per, 3)) / 8.0
                for fx, fy, fz in f:
                    pts.append(((x + fx) * EDGE_LEAF, (y + fy) * EDGE_LEAF, (z + fz) * EDGE_LEAF, 1.0))
    return pts


def edge_cases():
    """Hand-made exported clouds -> {name: (points N x 4 fp32 at EDGE_LEAF, viewpoint, variant)}, where `variant` is
    the deliberately wrong restatement (keyword arguments of normals()) that changes the answer on that case; None
    for the empty map, on which nothing can differ."""
    rng = np.random.RandomState(7)
    wrap = {"neighbour_fn": naive_neighbour}
    cases = {}
    # the last x index of rows y0, y0 + 1 beside the first x index of rows y0 + 1, y0 + 2 (naive: x + 1 wraps to the
    # next row's first voxel)
    pts = _block([LAST - 1, LAST], [5, 6], [-3, -2], rng) + _block([-HALF, -HALF + 1], [6, 7], [-3, -2], rng)
    cases["x_wrap_into_next_row"] = (pts, (0.0, 0.0, 0.0), wrap)
    # the last y index of plane z0 beside the first y index of plane z0 + 1
    pts = _block([40, 41], [LAST - 1, LAST], [9], rng) + _block([40, 41, 42], [-HALF, -HALF + 1], [10], rng)
    cases["y_wrap_into_next_plane"] = (pts, (1e3, -2e3, 5.0), wrap)
    # the last z plane (z + 1 leaves the key), with the x wrap inside it
    pts = (_block([LAST - 1, LAST], [-HALF, -HALF + 1], [LAST - 1, LAST], rng) +
           _block([-HALF, -HALF + 1], [-HALF + 1, -HALF + 2], [LAST], rng) + _block([0, 1], [LAST], [LAST], rng))
    cases["last_z_index"] = (pts, (0.0, 0.0, 0.0), wrap)
    # a lone voxel, two voxels (k = 2: NaN, unlike with a threshold of k < 2) and three collinear voxels (rank 1) with
    # the viewpoint exactly on the middle centroid (flip product exactly 0: no flip, unlike with <=)
    mid = (201.5 * EDGE_LEAF, 0.5 * EDGE_LEAF, -0.5 * EDGE_LEAF)
    pts = [(0.25, 0.25, 0.25, 1.0), (100.5 * EDGE_LEAF, 0.25, 0.25, 1.0), (101.5 * EDGE_LEAF, 0.25, 0.25, 1.0)]
    pts += [((200.5 + i) * EDGE_LEAF, mid[1], mid[2], 1.0) for i in range(3)]
    cases["lone_pair_collinear"] = (pts, mid, [{"min_k": 2}, {"flip_le": True}])
    cases["empty"] = ([], (0.0, 0.0, 0.0), None)
    return {k: (np.array(p, np.float32).reshape(-1, 4), vp, var) for k, (p, vp, var) in cases.items()}


def naive_neighbour(keys, vox, off):
    """WRONG on purpose (sensitivity tests): key + offset arithmetic on the packed key, which wraps across rows and
    planes at the edges of the key range."""
    dx, dy, dz = off
    step = (dx + (dy << 21) + (dz << 42)) % (1 << 64)  # two's complement of a negative offset: the add wraps mod 2^64
    return np.asarray(keys, np.uint64) + np.uint64(step), np.ones(len(keys), bool)
