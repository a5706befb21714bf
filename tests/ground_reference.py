"""numpy restatement of the ground of the whole-run voxel map (csrc/densemap.cuh dense_ground_*; include/loam_b200.h
"Ground of the whole-run voxel map").  y is up.

  * candidate: normal_x not NaN, (double)|n_y| >= cos(max_slope_deg * pi / 180) in double, and n_w <= max_curvature in
    fp32 unless max_curvature is +inf (a NaN w fails);
  * the candidates compacted in key order (a sorted key array stays sorted); candidate pairs: the box of
    segment_reference.candidate_pairs at r = floor(max(tol, max_step) / leaf) + 1;
  * edge: dx*dx + dz*dz <= tol^2 and |dy| <= max_step in fp64 of the float centroids;
  * patches: components of size >= min_size, ranked and recorded as segment_reference does, with target indices as the
    entry indices; the ground flags: the voxels of a patch;
  * above ground: segment_reference's Euclidean segmentation over the target voxels that are not ground;
  * cloud: q = pointAssociateToMap(pose, p) and align_reference.search over the ground voxels only; ground when a match
    has |pd| <= max_height, pd = (nx*(qx - cx) + ny*(qy - cy)) + nz*(qz - cz) in fp32; -1 for a point that is not
    finite or whose q lies outside the key range.

`variant` selects a deliberately wrong restatement (tests/test_ground_reference.py must catch each one): "dist3d" the
3-D distance instead of the horizontal one; "signed_ny" n_y without the absolute value; "no_curvature" the curvature
test dropped; "match_all" the cloud's match over every voxel with a normal; "height_strict" |pd| < max_height.
"""
import math

import numpy as np

import align_reference as ar
import dense_reference as dr
import map_reference as mr
import segment_reference as sr

F = np.float32
VARIANTS = ("dist3d", "signed_ny", "no_curvature", "match_all", "height_strict")


class Params:
    def __init__(self, max_slope_deg=15.0, max_curvature=0.05, tol=0.3, max_step=0.2, min_size=200):
        self.max_slope_deg = F(max_slope_deg)
        self.max_curvature = F(max_curvature)
        self.tol = F(tol)
        self.max_step = F(max_step)
        self.min_size = int(min_size)

    def ctypes(self):
        from loam_velodyne_b200 import api
        return api.GroundParams(self.max_slope_deg, self.max_curvature, self.tol, self.max_step, self.min_size)


def candidates(nrm, prm, variant=None):
    n = np.ascontiguousarray(nrm, np.float32).reshape(-1, 4)
    cos_max = math.cos(float(prm.max_slope_deg) * math.pi / 180.0)
    ny = n[:, 1] if variant == "signed_ny" else np.abs(n[:, 1])
    with np.errstate(invalid="ignore"):
        ok = ~np.isnan(n[:, 0]) & (ny.astype(np.float64) >= cos_max)
        if not np.isinf(prm.max_curvature) and variant != "no_curvature":
            ok &= n[:, 3] <= prm.max_curvature
    return ok


def radius_of(prm, leaf):
    return int(np.floor(max(float(prm.tol), float(prm.max_step)) / float(F(leaf)))) + 1


def ground_edges(ckeys, cpos, prm, leaf, variant=None):
    """Edges (i, j), i < j, between compacted positions of the candidates."""
    ii, jj = sr.candidate_pairs(ckeys, radius_of(prm, leaf))
    d = cpos[ii, :3].astype(np.float64) - cpos[jj, :3].astype(np.float64)
    if variant == "dist3d":
        h = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    else:
        h = d[:, 0] * d[:, 0] + d[:, 2] * d[:, 2]
    t = float(prm.tol)
    e = (h <= t * t) & (np.abs(d[:, 1]) <= float(prm.max_step))
    return ii[e], jj[e]


def _segment_subset(n_target, sel, ckeys, cpos, ii, jj, min_size, max_size):
    """segment_reference's components, ranks and records over the selected target voxels (compacted in key order, entry
    index = target index) with the given edges -> (labels int32[n_target], records)."""
    orig = np.nonzero(sel)[0]
    m = orig.size
    labels = np.full(n_target, -1, np.int32)
    if m == 0:
        return labels, sr._records(None, None, None, 0, np.zeros(0), np.zeros(0))
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    _, cc = connected_components(coo_matrix((np.ones(ii.size, np.int8), (ii, jj)), shape=(m, m)), directed=False)
    root_of_cc = np.full(cc.max() + 1, m, np.int64)
    np.minimum.at(root_of_cc, cc, np.arange(m))
    root = root_of_cc[cc]
    size = np.zeros(m, np.int64)
    np.add.at(size, root, 1)
    first = np.full(m, sr.INT_MAX, np.int64)
    np.minimum.at(first, root, orig)
    roots = np.nonzero(size > 0)[0]
    kept = roots[(size[roots] >= min_size) & (size[roots] <= max_size)]
    kept = kept[np.lexsort((first[kept], -size[kept]))]
    segid = np.full(m, -1, np.int64)
    segid[kept] = np.arange(kept.size)
    lab = segid[root]
    labels[orig] = lab
    return labels, sr._records(lab, orig, cpos, kept.size, size[kept], first[kept])


def dense_ground(keys, cent, nrm, leaf, prm, variant=None):
    """A target (ascending keys, centroids, normals) -> (labels int32[N], patches dict, ground bool[N])."""
    keys = np.asarray(keys, np.uint64)
    cent = np.ascontiguousarray(cent, np.float32).reshape(-1, 4)
    cand = candidates(nrm, prm, variant)
    ck, cp = keys[cand], cent[cand]
    ii, jj = ground_edges(ck, cp, prm, leaf, variant)
    labels, seg = _segment_subset(keys.size, cand, ck, cp, ii, jj, prm.min_size, sr.INT_MAX)
    return labels, seg, labels >= 0


def segment_above_ground(keys, cent, leaf, ground, tol, min_size=1, max_size=sr.INT_MAX):
    """dense_segment over the voxels that are not ground -> (labels int32[N], -1 on the ground; segments dict)."""
    keys = np.asarray(keys, np.uint64)
    cent = np.ascontiguousarray(cent, np.float32).reshape(-1, 4)
    sel = ~np.asarray(ground, bool)
    ck, cp = keys[sel], cent[sel]
    ii, jj = sr.edges(ck, cp, tol, leaf)
    return _segment_subset(keys.size, sel, ck, cp, ii, jj, min_size, max_size)


def ground_cloud(target, ground, pts, twist6, search_radius, max_height, variant=None):
    """A sensor-frame cloud at twist6 against an align_reference.Target and its ground flags -> (labels int8[N],
    the points labelled 0 in input order)."""
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
    finite = np.isfinite(p[:, :3]).all(axis=1)
    with np.errstate(invalid="ignore", over="ignore"):
        q = mr.Pose(twist6).to_map(np.where(finite[:, None], p, F(0.0)))
    q[~finite] = np.nan
    nrm = target.nrm
    if variant != "match_all":
        nrm = nrm.copy()
        nrm[~np.asarray(ground, bool), 0] = np.nan  # only ground voxels are admitted
    match = ar.search(ar.Target(target.leaf, target.keys, target.cent, nrm), q, search_radius)
    labels = np.where(dr.voxel_keys(q, target.leaf) != dr.EMPTY, 0, -1).astype(np.int8)
    has = np.nonzero(match >= 0)[0]
    if has.size:
        c, nv, qh = target.cent[match[has]], target.nrm[match[has]], q[has]
        pd = (nv[:, 0] * (qh[:, 0] - c[:, 0]) + nv[:, 1] * (qh[:, 1] - c[:, 1])) + nv[:, 2] * (qh[:, 2] - c[:, 2])
        h = F(max_height)
        on = np.abs(pd) < h if variant == "height_strict" else np.abs(pd) <= h
        labels[has[on]] = 1
    return labels, p[labels == 0]


def brute_ground_edges(cent, cand, prm):
    """Every candidate pair i < j (target indices) with the ground edge, O(n^2) over all pairs."""
    idx = np.nonzero(cand)[0]
    q = np.ascontiguousarray(cent, np.float32).reshape(-1, 4)[idx, :3].astype(np.float64)
    d = q[:, None, :] - q[None, :, :]
    h = d[..., 0] * d[..., 0] + d[..., 2] * d[..., 2]
    t = float(prm.tol)
    e = np.triu((h <= t * t) & (np.abs(d[..., 1]) <= float(prm.max_step)), 1)
    i, j = np.nonzero(e)
    return set(zip(idx[i].tolist(), idx[j].tolist()))
