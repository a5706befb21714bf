"""numpy restatement of the Euclidean segmentation (csrc/densemap.cuh dense_seg_*; include/loam_b200.h "Euclidean
segmentation of the whole-run voxel map and of clouds").

  * entries: a target's voxels in ascending key order (keys and centroids as the target holds them), or a cloud's
    points keyed by dense_reference.voxel_keys at cell = tol and sorted stably (skipped points last, not entries);
  * candidates: per (z, y) row offset of the box at r = floor(tol / cell) + 1, a searchsorted of the row's first and
    last key over the sorted keys, x clamped to the key range and rows outside it skipped (never wrapping);
  * edge: d2 = (dx*dx + dy*dy) + dz*dz in fp64 of the float coordinates, d2 <= tol^2 in fp64;
  * components with scipy, each named by its smallest sorted position; size, smallest entry index, the filter, the
    rank (size descending, smallest entry index ascending);
  * records: float min / max (the first member in entry order that reaches the extreme gives the sign of a zero) and
    the fp64 sums of the members in ascending entry index, chunks of 256 summed one by one from 0.0, the chunk sums
    added in chunk order from 0.0; centroid (float32)(sum / size).

`variant` selects a deliberately wrong restatement (tests/test_segment_reference.py must catch each one):
  "r_minus_1" a box one voxel smaller; "strict" d2 < tol^2; "fp32" distances in float32; "tie_largest" ties ranked by
  the largest member index; "no_filter" non-finite and out-of-range points keyed by a clamped voxel instead of skipped.
A box walk that wraps rows is not among them: a wrapped row only adds candidates about 2^21 voxels away, which the
edge test rejects, so it cannot change any output.
"""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

import dense_reference as dr

CHUNK = 256
AXIS = 1 << 21
INT_MAX = 2**31 - 1
VARIANTS = ("r_minus_1", "strict", "fp32", "tie_largest", "no_filter")


def _keys_no_filter(p, cell):
    inv = np.float32(1.0) / np.float32(cell)
    with np.errstate(invalid="ignore", over="ignore"):
        f = np.floor(p[:, :3] * inv)
    f = np.nan_to_num(f, nan=0.0, posinf=dr.LIM - 1, neginf=-dr.LIM)
    v = (np.clip(f, -dr.LIM, dr.LIM - 1).astype(np.int64) + dr.HALF).astype(np.uint64)
    return (v[:, 2] << np.uint64(42)) | (v[:, 1] << np.uint64(21)) | v[:, 0]


def radius_of(tol, cell):
    return int(np.floor(float(np.float32(tol)) / float(np.float32(cell)))) + 1


def candidate_pairs(skeys, r):
    """(i, j), j > i, of the sorted keys (DENSE_EMPTY entries excluded) whose voxels lie within r of each other per
    axis, as dense_box_walk finds them."""
    m = int(np.count_nonzero(skeys != dr.EMPTY))
    k = skeys[:m]
    u = dr.key_voxel(k) + dr.HALF
    idx = np.arange(m)
    x0 = np.maximum(u[:, 0] - r, 0).astype(np.uint64)
    x1 = np.minimum(u[:, 0] + r, AXIS - 1).astype(np.uint64)
    ii, jj = [], []
    for dz in range(-r, r + 1):
        z = u[:, 2] + dz
        for dy in range(-r, r + 1):
            y = u[:, 1] + dy
            ok = (z >= 0) & (z < AXIS) & (y >= 0) & (y < AXIS)
            row = (np.where(ok, z, 0).astype(np.uint64) << np.uint64(42)) | \
                  (np.where(ok, y, 0).astype(np.uint64) << np.uint64(21))
            lo = np.maximum(np.searchsorted(k, row | x0, "left"), idx + 1)
            hi = np.searchsorted(k, row | x1, "right")
            cnt = np.where(ok, np.maximum(hi - lo, 0), 0)
            tot = int(cnt.sum())
            if tot == 0:
                continue
            rep = np.repeat(idx, cnt)
            off = np.arange(tot) - np.repeat(np.cumsum(cnt) - cnt, cnt)
            ii.append(rep)
            jj.append(np.repeat(lo, cnt) + off)
    if not ii:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(ii), np.concatenate(jj)


def edge_mask(spos, ii, jj, tol, variant=None):
    if variant == "fp32":
        d = spos[ii, :3] - spos[jj, :3]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        t = np.float32(tol)
        return d2 <= t * t
    d = spos[ii, :3].astype(np.float64) - spos[jj, :3].astype(np.float64)
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    t = float(np.float32(tol))
    return d2 < t * t if variant == "strict" else d2 <= t * t


def edges(skeys, spos, tol, cell, variant=None):
    """Edges (i, j), i < j, between sorted positions."""
    r = radius_of(tol, cell) - (1 if variant == "r_minus_1" else 0)
    ii, jj = candidate_pairs(skeys, r)
    e = edge_mask(spos, ii, jj, tol, variant)
    return ii[e], jj[e]


def _segment(skeys, spos, orig, tol, cell, min_size, max_size, variant):
    n = skeys.size
    if n == 0:
        return np.zeros(0, np.int32), _records(None, None, None, 0, np.zeros(0), np.zeros(0))
    valid = skeys != dr.EMPTY
    ii, jj = edges(skeys, spos, tol, cell, variant)
    g = coo_matrix((np.ones(ii.size, np.int8), (ii, jj)), shape=(n, n))
    _, cc = connected_components(g, directed=False)
    root_of_cc = np.full(cc.max() + 1, n, np.int64)
    np.minimum.at(root_of_cc, cc, np.arange(n))
    root = np.where(valid, root_of_cc[cc], -1)
    ent = orig if orig is not None else np.arange(n)
    size = np.zeros(n, np.int64)
    first = np.full(n, INT_MAX, np.int64)
    last = np.full(n, -1, np.int64)
    np.add.at(size, root[valid], 1)
    np.minimum.at(first, root[valid], ent[valid])
    np.maximum.at(last, root[valid], ent[valid])
    roots = np.nonzero(size > 0)[0]
    kept = roots[(size[roots] >= min_size) & (size[roots] <= max_size)]
    tie = last[kept] if variant == "tie_largest" else first[kept]
    kept = kept[np.lexsort((tie, -size[kept]))]
    segid = np.full(n, -1, np.int64)
    segid[kept] = np.arange(kept.size)
    lab_sorted = np.where(valid, segid[np.maximum(root, 0)], -1)
    labels = np.full(n, -1, np.int32)
    labels[ent] = lab_sorted
    return labels, _records(lab_sorted, ent, spos, kept.size, size[kept], first[kept])


def _records(lab_sorted, ent, spos, K, size, first):
    out = {"size": size.astype(np.int32), "first": first.astype(np.int32),
           "lo": np.zeros((K, 3), np.float32), "hi": np.zeros((K, 3), np.float32),
           "centroid": np.zeros((K, 3), np.float32)}
    if K == 0:
        return out
    mem = np.nonzero(lab_sorted >= 0)[0]
    mem = mem[np.lexsort((ent[mem], lab_sorted[mem]))]  # by segment, then entry index
    s = lab_sorted[mem]
    start = np.searchsorted(s, np.arange(K))
    t = np.arange(mem.size) - start[s]
    vals = spos[mem, :3]
    # min / max: the first member in entry order reaching the extreme
    for name, red in (("lo", np.minimum), ("hi", np.maximum)):
        ext = red.reduceat(vals, start, axis=0)
        for a in range(3):
            e = ext[s, a]
            eq = np.nonzero((vals[:, a] == e) | (np.isnan(vals[:, a]) & np.isnan(e)))[0]
            _, at = np.unique(s[eq], return_index=True)
            out[name][:, a] = vals[eq[at], a]
    # chunked fp64 sums
    cid = np.cumsum(np.concatenate([[0], (t[1:] % CHUNK == 0) | (s[1:] != s[:-1])]))
    v64 = vals.astype(np.float64)
    csum = np.zeros((cid[-1] + 1, 3), np.float64)
    pos = t % CHUNK
    for j in range(CHUNK):
        sel = pos == j
        if not sel.any():
            break
        csum[cid[sel]] = csum[cid[sel]] + v64[sel]
    head = np.concatenate([[True], cid[1:] != cid[:-1]])
    cs, ci = s[head], t[head] // CHUNK
    tot = np.zeros((K, 3), np.float64)
    for j in range(int(ci.max()) + 1):
        sel = ci == j
        tot[cs[sel]] = tot[cs[sel]] + csum[sel]
    out["centroid"] = (tot / size[:, None].astype(np.float64)).astype(np.float32)
    return out


def target_segment(keys, cent, leaf, tol, min_size=1, max_size=INT_MAX, variant=None):
    """A target's keys (ascending) and centroids in the same order -> (labels int32[N], segments dict)."""
    return _segment(np.asarray(keys, np.uint64), np.ascontiguousarray(cent, np.float32).reshape(-1, 4), None, tol,
                    leaf, min_size, max_size, variant)


def cloud_segment(pts, tol, min_size=1, max_size=INT_MAX, variant=None):
    """A cloud's points -> (labels int32[N] in input order, segments dict)."""
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
    k = _keys_no_filter(p, tol) if variant == "no_filter" else dr.voxel_keys(p, tol)
    order = np.argsort(k, kind="stable")
    return _segment(k[order], p[order], order, tol, tol, min_size, max_size, variant)


def target_of(pts, leaf):
    """(keys ascending, centroids in that order) of points loaded as a target (one per voxel)."""
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
    k = dr.voxel_keys(p, leaf)
    o = np.argsort(k, kind="stable")
    return k[o], p[o]


def brute_edges(pts, tol):
    """Every pair i < j of finite, in-range points with fp64 d2 <= tol^2 (O(n^2)), as input indices."""
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
    ok = np.nonzero(dr.voxel_keys(p, tol) != dr.EMPTY)[0]
    q = p[ok, :3].astype(np.float64)
    d = q[:, None, :] - q[None, :, :]
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    t = float(np.float32(tol))
    i, j = np.nonzero(np.triu(d2 <= t * t, 1))
    return set(zip(ok[i].tolist(), ok[j].tolist()))


def cloud_edges(pts, tol, variant=None):
    """The restatement's edges of a cloud as input-index pairs (i < j)."""
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
    k = dr.voxel_keys(p, tol)
    order = np.argsort(k, kind="stable")
    ii, jj = edges(k[order], p[order], tol, tol, variant)
    a, b = order[ii], order[jj]
    return set(zip(np.minimum(a, b).tolist(), np.maximum(a, b).tolist()))
