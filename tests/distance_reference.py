"""Numpy restatement of the distance field of the whole-run voxel map (include/loam_b200.h "Distance field of the
whole-run voxel map"; csrc/densemap.cuh: dense_edt_*_kernel, dense_distance_query_kernel).

Field: occupied = a voxel whose key is in the target; the box is the voxels lo + [0, dims), numpy shape (nz, ny, nx);
sq = the squared Euclidean distance in voxel units from a cell to the nearest occupied voxel of the whole target,
computed exactly over the box grown by pad = floor(max_distance / L) + 1 voxels per side; beyond (sqrt(sq) * L >
max_distance): sq = -1, dist = +inf; otherwise dist = float32(sqrt(sq) * L).

Query: fp64 without FMA in the header's expression order (numpy rounds every operation on its own), one rounding to
float32 at the end.

The keyword arguments of field() and query() are deliberately wrong restatements, each of which some case of
tests/test_distance_reference.py must catch: pad_floor (pad = floor(R) without the + 1), beyond_ge (>= in the beyond
test), ignore_outside (obstacles outside the box ignored) and hull_off_by_one (queries defined up to g_a <= n_a).

pad = floor(R) alone (R = max_distance / L in double) would already give the same values: an obstacle k voxels away
along an axis is within range only if k L <= max_distance, and k L is exact in double, so the correctly rounded R is
then >= k.  The + 1 keeps the claim free of that rounding argument; what it changes is which boxes fit the limits, so
pad_floor is caught by box_ok()."""
import math

import numpy as np

import dense_reference as dr

INF = np.int64(1) << np.int64(40)  # no site on the line; never reached by a sum of squares of padded offsets


def edt_sq(occ):
    """Exact squared EDT (int64) of a boolean grid to its True cells, separable: per axis, the lower envelope of
    (i - j)^2 + f(j) by growing offsets, stopped once no offset can lower any value of a line that holds a site.  INF
    where the grid has no True cell."""
    f = np.where(np.asarray(occ, bool), np.int64(0), INF)
    for axis in range(f.ndim):
        f = _pass(f, axis)
    return f


def _pass(f, axis):
    g = np.moveaxis(f, axis, -1)
    m = g.shape[-1]
    has = np.broadcast_to((g < INF).any(axis=-1, keepdims=True), g.shape)
    best = g.copy()
    for d in range(1, m):
        live = best[has]
        if live.size == 0 or live.max() <= d * d:
            break
        dd = np.int64(d * d)
        np.minimum(best[..., d:], g[..., :-d] + dd, out=best[..., d:])
        np.minimum(best[..., :-d], g[..., d:] + dd, out=best[..., :-d])
    best = np.minimum(best, INF)
    return np.moveaxis(best, -1, axis)


def target_voxels(keys):
    """(M, 3) int64 voxel indices (x, y, z) of target keys."""
    return dr.key_voxel(np.asarray(keys, np.uint64)).astype(np.int64).reshape(-1, 3)


def occupancy(vox, lo, dims):
    """Boolean grid (nz, ny, nx) of the voxels lo + [0, dims) that hold a target voxel."""
    lo = np.asarray(lo, np.int64).reshape(3)
    dims = np.asarray(dims, np.int64).reshape(3)
    occ = np.zeros(tuple(int(d) for d in dims[::-1]), bool)
    r = vox - lo
    ok = ((r >= 0) & (r < dims)).all(axis=1)
    r = r[ok]
    occ[r[:, 2], r[:, 1], r[:, 0]] = True
    return occ


def pad_of(leaf, max_distance, pad_floor=False):
    R = float(np.float32(max_distance)) / float(np.float32(leaf))
    return int(math.floor(R)) + (0 if pad_floor else 1)


MAX_RATIO, MAX_AXIS, MAX_CELLS, HALF = 1024, 8192, 1 << 27, 1 << 20


def box_ok(leaf, lo, dims, max_distance, pad_floor=False):
    """Whether loam_b200_dense_distance_build accepts the box (LOAM_B200_ERR_ARG otherwise): finite max_distance > 0,
    max_distance / L <= 1024, dims >= 1, every padded axis <= 8192, padded cells <= 2^27, the padded box inside the
    key range [-2^20, 2^20)."""
    md = float(np.float32(max_distance))
    if not (math.isfinite(md) and md > 0.0) or any(int(d) < 1 for d in dims):
        return False
    if not md / float(np.float32(leaf)) <= MAX_RATIO:
        return False
    pad = pad_of(leaf, max_distance, pad_floor)
    n = [int(d) + 2 * pad for d in dims]
    plo = [int(v) - pad for v in lo]
    return (max(n) <= MAX_AXIS and n[0] * n[1] * n[2] <= MAX_CELLS and min(plo) >= -HALF and
            max(a + b for a, b in zip(plo, n)) <= HALF)


def field(keys, leaf, lo, dims, max_distance, pad_floor=False, beyond_ge=False, ignore_outside=False):
    """-> (dist float32, sq int32), each (nz, ny, nx), of the target's keys."""
    L = float(np.float32(leaf))
    md = float(np.float32(max_distance))
    pad = 0 if ignore_outside else pad_of(leaf, max_distance, pad_floor)
    lo = np.asarray(lo, np.int64).reshape(3)
    dims = np.asarray(dims, np.int64).reshape(3)
    occ = occupancy(target_voxels(keys), lo - pad, dims + 2 * pad)
    s = edt_sq(occ)[pad:pad + dims[2], pad:pad + dims[1], pad:pad + dims[0]]
    w = np.sqrt(np.minimum(s, INF - 1).astype(np.float64)) * L
    beyond = (s >= INF) | ((w >= md) if beyond_ge else (w > md))
    sq = np.where(beyond, -1, s).astype(np.int32)
    dist = np.where(beyond, np.float32(np.inf), w.astype(np.float32)).astype(np.float32)
    return dist, sq


def _lerp(a, b, f):
    return a + f * (b - a)


def query(sq, leaf, lo, max_distance, pts, hull_off_by_one=False):
    """The field sq (nz, ny, nx) of the box at lo, queried at map-frame pts (N x 4) -> (dist float32[N],
    grad float32[N, 3])."""
    L = float(np.float32(leaf))
    md = float(np.float32(max_distance))
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)[:, :3].astype(np.float64)
    n = np.array(sq.shape[::-1], np.int64)
    lo = np.asarray(lo, np.int64).reshape(3)
    with np.errstate(invalid="ignore"):
        g = (p / L - 0.5) - lo.astype(np.float64)
        hi = n.astype(np.float64) if hull_off_by_one else (n - 1).astype(np.float64)
        ok = ((n >= 2) & (g >= 0.0) & (g <= hi)).all(axis=1)
    gs = np.where(ok[:, None], g, 0.0)
    i = np.minimum(np.floor(gs).astype(np.int64), np.maximum(n - 2, 0))
    f = gs - i
    w = np.where(sq < 0, md, np.sqrt(np.maximum(sq, 0).astype(np.float64)) * L)
    nz, ny, nx = sq.shape

    def c(dx, dy, dz):
        x = np.minimum(i[:, 0] + dx, nx - 1)
        y = np.minimum(i[:, 1] + dy, ny - 1)
        z = np.minimum(i[:, 2] + dz, nz - 1)
        return w[z, y, x]

    w000, w100, w010, w110 = c(0, 0, 0), c(1, 0, 0), c(0, 1, 0), c(1, 1, 0)
    w001, w101, w011, w111 = c(0, 0, 1), c(1, 0, 1), c(0, 1, 1), c(1, 1, 1)
    fx, fy, fz = f[:, 0], f[:, 1], f[:, 2]
    d = _lerp(_lerp(_lerp(w000, w100, fx), _lerp(w010, w110, fx), fy),
              _lerp(_lerp(w001, w101, fx), _lerp(w011, w111, fx), fy), fz)
    gx = _lerp(_lerp(w100 - w000, w110 - w010, fy), _lerp(w101 - w001, w111 - w011, fy), fz) / L
    gy = _lerp(_lerp(w010 - w000, w110 - w100, fx), _lerp(w011 - w001, w111 - w101, fx), fz) / L
    gz = _lerp(_lerp(w001 - w000, w101 - w100, fx), _lerp(w011 - w010, w111 - w110, fx), fy) / L
    dist = np.where(ok, d, np.nan).astype(np.float32)
    grad = np.where(ok[:, None], np.stack([gx, gy, gz], axis=1), np.nan).astype(np.float32)
    return dist, grad


def centres(leaf, vox):
    """Map-frame float32 points (N x 4) at the centres of voxels vox (N x 3): (v + 0.5) * leaf in float32."""
    v = np.asarray(vox, np.float64).reshape(-1, 3)
    p = ((v + 0.5) * float(np.float32(leaf))).astype(np.float32)
    return np.ascontiguousarray(np.concatenate([p, np.zeros((p.shape[0], 1), np.float32)], axis=1))


def keys_of_voxels(vox):
    """Target keys of integer voxels (N x 3, x y z) by the key codec."""
    v = np.asarray(vox, np.int64).reshape(-1, 3) + dr.HALF
    return ((v[:, 2].astype(np.uint64) << np.uint64(42)) | (v[:, 1].astype(np.uint64) << np.uint64(21)) |
            v[:, 0].astype(np.uint64))


def edge_cases():
    """{name: (leaf, voxels M x 3, lo, dims, max_distance)}: hand-made targets for the GPU (loaded from voxel centres)
    and for the wrong restatements."""
    c = {}
    c["lone"] = (0.2, [[3, -2, 5]], (-4, -9, -2), (15, 14, 13), 1.0)
    # voxels on the faces and corners of 8^3 bricks (key bias 2^20 is a multiple of 8, so voxel 0 starts a brick)
    c["brick_faces"] = (0.1, [[7, 0, 0], [8, 0, 0], [0, 7, 8], [-1, -1, -1], [-8, 15, 16], [15, -9, 7]],
                        (-12, -12, -12), (30, 29, 31), 0.75)
    c["negative"] = (0.25, [[-100, -37, -64], [-97, -40, -61]], (-110, -45, -70), (20, 12, 16), 2.0)
    c["pad_only"] = (0.1, [[-3, 2, 2]], (0, 0, 0), (6, 5, 4), 0.3)  # the only obstacle 3 voxels outside the box
    c["exact_range"] = (0.5, [[0, 0, 0]], (2, 0, 0), (4, 1, 1), 1.0)  # a cell at exactly max_distance
    c["thin_x"] = (0.2, [[0, 0, 0], [2, 5, -3]], (1, -4, -6), (1, 9, 11), 1.2)
    c["thin_y"] = (0.2, [[0, 0, 0], [2, 5, -3]], (-4, 1, -6), (9, 1, 11), 1.2)
    c["thin_z"] = (0.2, [[0, 0, 0], [2, 5, -3]], (-4, -6, 1), (9, 11, 1), 1.2)
    c["one_cell"] = (0.3, [[1, 1, 1]], (0, 0, 0), (1, 1, 1), 0.9)
    c["wall"] = (0.1, [[x, y, 4] for x in range(-6, 7) for y in range(-3, 4)], (-8, -5, -3), (17, 11, 14), 0.5)
    return c
