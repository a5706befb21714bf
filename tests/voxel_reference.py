"""Plain restatements of the shared radix sort, the voxel grid filter and the mapping stage's stack round trip, for
the tests (numpy only).

- sort_pairs: radix_sort_pairs (csrc/loam_b200.cu) -- 8 bits per pass, at most four passes, an even number of passes
  for callers that read the first buffer directly; the result is a stable sort on the bits those passes cover.
- voxel_grid: the product's VoxelGrid semantics (csrc/voxel.cuh), every operation in float32: bounding box, the int32
  overflow guard on the truncated extents, origin and extents from floor(min * inv) / floor(max * inv), a wrapping
  int32 linear voxel key, a stable sort by key, and per voxel the sequential float32 sum of its points in input order
  divided by the count.  Sums are sequential on purpose: np.sum and np.add.reduceat sum float32 pairwise and differ.
- stack_roundtrip: pointAssociateToMap then pointAssociateTobeMapped with the predicted pose, in the operation order of
  stack_roundtrip (csrc/mapping_lm.cuh).
"""
from __future__ import annotations

import numpy as np

from map_reference import Pose

F = np.float32
INT32_MAX = 2**31 - 1
RS_MAX_PASSES = 4
SEQ_LOOP_MAX = 32  # runs up to this long are summed by a loop over the position in the run, longer ones by cumsum


def sort_passes(key_bits, out_params=True):
    passes = min((int(key_bits) + 7) // 8, RS_MAX_PASSES)
    if not out_params and passes % 2:
        passes += 1
    return passes


def sort_pairs(keys, vals, key_bits, out_params=True):
    """(keys, vals) sorted stably by the low 8 * passes bits of the keys."""
    keys = np.asarray(keys, np.uint32)
    vals = np.asarray(vals)
    mask = np.uint64((1 << (8 * sort_passes(key_bits, out_params))) - 1)
    order = np.argsort(keys.astype(np.uint64) & mask, kind="stable")
    return keys[order], vals[order]


def voxel_meta(pts, leaf):
    """(inv, minb[3], div[3], overflow) of the cloud's bounding box, as voxel_meta_from_bbox computes them."""
    p = np.asarray(pts, F).reshape(-1, 4)
    inv = F(1) / F(leaf)
    mn = p[:, :3].min(axis=0)
    mx = p[:, :3].max(axis=0)
    ext = ((mx - mn) * inv).astype(np.int64) + 1
    overflow = int(ext[0]) * int(ext[1]) * int(ext[2]) > INT32_MAX
    minb = np.floor(mn * inv).astype(np.int64)
    div = np.floor(mx * inv).astype(np.int64) - minb + 1
    return inv, minb, div, overflow


def voxel_keys(pts, inv, minb, div):
    """uint32 linear voxel key of every point (int32 arithmetic, wrapping)."""
    p = np.asarray(pts, F).reshape(-1, 4)
    ijk = [(np.floor(p[:, a] * inv) - F(minb[a])).astype(np.int32).astype(np.int64) for a in range(3)]
    key = ijk[0] + ijk[1] * int(div[0]) + ijk[2] * int(div[0]) * int(div[1])
    return (key & 0xFFFFFFFF).astype(np.uint32)


def run_sums(q, heads, counts):
    """Sequential float32 sum of every run q[h : h + c], first element first."""
    sums = np.zeros((heads.shape[0], q.shape[1]), F)
    short = counts <= SEQ_LOOP_MAX
    for j in range(int(min(counts.max(initial=0), SEQ_LOOP_MAX))):
        live = short & (counts > j)
        sums[live] += q[heads[live] + j]
    for r in np.flatnonzero(~short):
        h, c = int(heads[r]), int(counts[r])
        sums[r] = np.cumsum(q[h:h + c], axis=0, dtype=F)[-1]
    return sums


def voxel_grid(pts, leaf):
    """Centroid per occupied voxel, ascending voxel key; the input unchanged when the guard trips."""
    p = np.asarray(pts, F).reshape(-1, 4)
    if p.shape[0] == 0:
        return p.copy()
    inv, minb, div, overflow = voxel_meta(p, leaf)
    if overflow:
        return p.copy()
    key = voxel_keys(p, inv, minb, div)
    order = np.argsort(key, kind="stable")
    ks, q = key[order], p[order]
    heads = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    counts = np.diff(np.r_[heads, ks.shape[0]])
    return run_sums(q, heads, counts) / counts.astype(F)[:, None]


# clouds at leaf 1.0 spanning the two corners: extents 1024 x 1024 x 2047 fit the guard, 1024 x 1024 x 2048 do not, and
# "wrap" fits it (extents 1024 x 1024 x 2047) with div 1025 x 1025 x 2048 = 2 151 680 000, so keys pass 2^31
GUARD_BOXES = {
    "fit": ((0.0, 0.0, 0.0), (1023.5, 1023.5, 2046.5)),
    "over": ((0.0, 0.0, 0.0), (1023.5, 1023.5, 2047.5)),
    "wrap": ((0.5, 0.5, 0.5), (1024.0, 1024.0, 2047.4)),
}


def guard_box_cloud(name, n=4096, seed=0):
    """n points inside the box (its two corners first), clustered eight to a voxel around random centres."""
    lo, hi = (np.asarray(c, F) for c in GUARD_BOXES[name])
    rng = np.random.RandomState(seed)
    m = (n - 2 + 7) // 8
    centres = np.floor(rng.uniform(lo, hi, (m, 3))).astype(F)
    xyz = np.repeat(centres, 8, axis=0)[:n - 2] + rng.uniform(0.0, 0.99, (n - 2, 3)).astype(F)
    xyz = np.clip(xyz, lo, hi)
    pts = np.empty((n, 4), F)
    pts[0, :3], pts[1, :3], pts[2:, :3] = lo, hi, xyz
    pts[:, 3] = rng.uniform(0.0, 100.0, n).astype(F)
    return pts


def pairwise_sum(q):
    """np.sum of every column as a 1-D array: pairwise above eight elements (np.sum over axis 0 of a 2-D array adds
    row by row, which is sequential)."""
    return np.array([np.sum(np.ascontiguousarray(q[:, j]), dtype=F) for j in range(q.shape[1])], F)


def _orders_differ(q):
    seq = np.cumsum(q, axis=0, dtype=F)[-1]
    rev = np.cumsum(q[::-1], axis=0, dtype=F)[-1]
    pair = pairwise_sum(q)
    return bool(np.any(seq != rev)) and (q.shape[0] < 128 or bool(np.any(seq != pair)))


ORDER_PROBE_LENGTHS = (3, 5, 17, 33, 300, 1500, 9000)


def order_probe_cloud(n_background, seed=0):
    """Voxels (leaf 1.0) whose float32 sums differ between sequential, reversed and pairwise order, scattered among
    n_background single points.  Runs of 1500 and 9000 points are longer than a 1024-key scan block and than any CTA's
    share of a one-cluster sort (<= 8192 keys), so they straddle those boundaries."""
    rng = np.random.RandomState(seed)
    parts = []
    for i, m in enumerate(ORDER_PROBE_LENGTHS):
        cell = np.array([3 * i - 7, 25 + i, 5 - 2 * i], F)  # above the background, coordinates of both signs
        while True:
            frac = rng.uniform(0.0, 0.999, (m, 4)).astype(F)
            frac[rng.rand(m) < 0.5] *= F(1e-3)  # mixed magnitudes
            q = np.empty((m, 4), F)
            q[:, :3] = cell + frac[:, :3]
            q[:, 3] = frac[:, 3] * F(100.0)
            if _orders_differ(q):
                break
        parts.append(q)
    bg = np.empty((n_background, 4), F)
    bg[:, :3] = rng.uniform(-20.0, 20.0, (n_background, 3)).astype(F)
    bg[:, 3] = rng.uniform(0.0, 100.0, n_background).astype(F)
    pts = np.concatenate(parts + [bg])
    return pts[rng.permutation(pts.shape[0])]


def stack_roundtrip(pts, twist6):
    """Stack points to the map frame and back into the sensor frame with the predicted pose (not an identity in fp32).
    The negated angles of pointAssociateTobeMapped flip the sine only."""
    pose = Pose(twist6)
    p = pose.to_map(pts)
    srx, sry, srz = pose.s
    crx, cry, crz = pose.c
    x = p[:, 0] - pose.pos[0]
    y = p[:, 1] - pose.pos[1]
    z = p[:, 2] - pose.pos[2]
    x1 = cry * x + (-sry) * z
    z1 = cry * z - (-sry) * x
    y2 = crx * y - (-srx) * z1
    z2 = (-srx) * y + crx * z1
    x3 = crz * x1 - (-srz) * y2
    y3 = (-srz) * x1 + crz * y2
    out = p.copy()
    out[:, 0], out[:, 1], out[:, 2] = x3, y3, z2
    return out
