"""Plain reference of the mapping stage's map bookkeeping (BasicLaserMapping.cpp:300-593), for the tests.

The map is what the reference holds: per kind, one point list per cube of the 21 x 11 x 21 grid.  Cubes are keyed
by their absolute cube coordinates (grid index minus the grid centre), so a roll of the grid only changes the centre
and drops the cubes that leave it.  Everything a pose touches is fp32 in the reference's operation order; the only
library call is the VoxelGrid filter, which the caller passes in (the checker's pcl::VoxelGrid).
"""
from __future__ import annotations

import numpy as np

from loam_velodyne_b200.api import sincos_f32

W, H, D = 21, 11, 21
DIMS = np.array([W, H, D], np.int64)
F = np.float32


def cube_ijk(pts, cen):
    """Grid indices (n x 3, possibly outside the grid) of map-frame points: the double-precision formula of :540-553,
    truncation toward zero and the decrement on the negative side."""
    v = np.asarray(pts, np.float32)[:, :3].astype(np.float64) + 25.0
    c = np.trunc(v / 50.0).astype(np.int64) + np.asarray(cen, np.int64)
    return c - (v < 0)


def in_grid(ijk):
    return np.all((ijk >= 0) & (ijk < DIMS), axis=1)


def grid_index(ijk):
    ijk = np.asarray(ijk, np.int64)
    return ijk[..., 0] + W * ijk[..., 1] + W * H * ijk[..., 2]


class Pose:
    """A twist (rot_x, rot_y, rot_z, x, y, z) with the sin / cos loam::Angle caches (glibc sinf / cosf)."""

    def __init__(self, twist6):
        t = np.asarray(twist6, np.float32).reshape(6)
        self.twist = t
        self.pos = t[3:].copy()
        sc = [sincos_f32(a) for a in t[:3]]
        self.s = [s for s, _ in sc]
        self.c = [c for _, c in sc]

    def to_map(self, pts):
        """pointAssociateToMap (:207-219) in the operation order of associate_to_map (csrc/mapping_lm.cuh)."""
        p = np.array(pts, np.float32, copy=True).reshape(-1, 4)
        srx, sry, srz = self.s
        crx, cry, crz = self.c
        x, y, z = p[:, 0], p[:, 1], p[:, 2]
        x1 = crz * x - srz * y
        y1 = srz * x + crz * y
        y2 = crx * y1 - srx * z
        z2 = srx * y1 + crx * z
        x3 = cry * x1 + sry * z2
        z3 = cry * z2 - sry * x1
        p[:, 0] = x3 + self.pos[0]
        p[:, 1] = y2 + self.pos[1]
        p[:, 2] = z3 + self.pos[2]
        return p


def window(twist6, cen):
    """Grid roll (:303-441) and field-of-view test (:443-500) at pose twist6 -> (new centre, valid cube indices,
    surround cube indices), both lists in the reference's i, j, k loop order."""
    pose = Pose(twist6)
    on_y = pose.to_map(np.array([[0.0, 10.0, 0.0, 0.0]], np.float32))[0, :3]
    cen = [int(c) for c in cen]
    centre = [int((float(pose.pos[a]) + 25.0) / 50.0) + cen[a] - (1 if float(pose.pos[a]) + 25.0 < 0 else 0)
              for a in range(3)]
    for a, dim in enumerate((W, H, D)):
        while centre[a] < 3:
            centre[a] += 1
            cen[a] += 1
        while centre[a] >= dim - 3:
            centre[a] -= 1
            cen[a] -= 1
    k10s3 = F(10.0) * F(np.sqrt(F(3.0)))
    valid, surround = [], []
    for i in range(centre[0] - 2, centre[0] + 3):
        for j in range(centre[1] - 2, centre[1] + 3):
            for k in range(centre[2] - 2, centre[2] + 3):
                if not (0 <= i < W and 0 <= j < H and 0 <= k < D):
                    continue
                cx, cy, cz = F(50.0) * F(i - cen[0]), F(50.0) * F(j - cen[1]), F(50.0) * F(k - cen[2])
                fov = False
                for ii in (-1, 1):
                    for jj in (-1, 1):
                        for kk in (-1, 1):
                            corner = np.array([cx + F(25.0) * F(ii), cy + F(25.0) * F(jj), cz + F(25.0) * F(kk)], F)
                            d1 = pose.pos - corner
                            d2 = on_y - corner
                            s1 = d1[0] * d1[0] + d1[1] * d1[1] + d1[2] * d1[2]
                            s2 = d2[0] * d2[0] + d2[1] * d2[1] + d2[2] * d2[2]
                            base = (F(100.0) + s1) - s2
                            r = k10s3 * F(np.sqrt(s1))
                            if base - r < 0 and base + r > 0:
                                fov = True
                idx = i + W * j + W * H * k
                if fov:
                    valid.append(idx)
                surround.append(idx)
    return tuple(cen), valid, surround


class CubeMap:
    """One kind (corner or surface) of the reference's cube clouds."""

    def __init__(self, cen=(10, 5, 10)):
        self.cen = tuple(int(c) for c in cen)
        self.cubes: dict[tuple, np.ndarray] = {}  # absolute cube coordinates -> points in insertion order

    def _key_of_index(self, idx):
        i, j, k = idx % W, (idx // W) % H, idx // (W * H)
        return (i - self.cen[0], j - self.cen[1], k - self.cen[2])

    def add(self, pts):
        """Append points (map frame) to their cubes in the given order; points outside the grid are dropped."""
        p = np.asarray(pts, np.float32).reshape(-1, 4)
        if p.shape[0] == 0:
            return
        ijk = cube_ijk(p, self.cen)
        keep = in_grid(ijk)
        p, ijk = p[keep], ijk[keep]
        gi = grid_index(ijk)
        order = np.argsort(gi, kind="stable")
        gi, p = gi[order], p[order]
        bounds = np.flatnonzero(np.diff(gi)) + 1
        for part_gi, part in zip(np.split(gi, bounds), np.split(p, bounds)):
            if part.shape[0] == 0:
                continue
            key = self._key_of_index(int(part_gi[0]))
            old = self.cubes.get(key)
            self.cubes[key] = part.copy() if old is None else np.concatenate([old, part])

    def roll_to(self, cen):
        """The grid centre moves; cubes that leave the 21 x 11 x 21 grid are cleared."""
        self.cen = tuple(int(c) for c in cen)
        c = np.asarray(self.cen, np.int64)
        self.cubes = {key: v for key, v in self.cubes.items()
                      if np.all((np.asarray(key) + c >= 0) & (np.asarray(key) + c < DIMS))}

    def cube(self, idx):
        return self.cubes.get(self._key_of_index(int(idx)), np.zeros((0, 4), np.float32))

    def from_map(self, valid):
        """laserCloud*FromMap (:503-509): the points of the valid cubes in list order."""
        parts = [self.cube(i) for i in valid]
        return np.concatenate(parts) if parts else np.zeros((0, 4), np.float32)

    def filter(self, valid, leaf, voxel_grid):
        """:580-593: every valid cube becomes VoxelGrid(its points)."""
        for idx in valid:
            key = self._key_of_index(int(idx))
            if key in self.cubes and self.cubes[key].shape[0]:
                self.cubes[key] = voxel_grid(self.cubes[key], leaf)

    def all_points(self):
        """Every cube's points, cubes in grid-index order (like the reference's cube array)."""
        c = np.asarray(self.cen, np.int64)
        keys = sorted(self.cubes, key=lambda a: int(grid_index(np.asarray(a) + c)))
        parts = [self.cubes[k] for k in keys]
        return np.concatenate(parts) if parts else np.zeros((0, 4), np.float32)

    def indices(self):
        c = np.asarray(self.cen, np.int64)
        return sorted(int(grid_index(np.asarray(k) + c)) for k in self.cubes if self.cubes[k].shape[0])


def sweep_update(maps, leaves, twist_predicted, twist_optimised, stacks_ds, voxel_grid):
    """One sweep of the map as process() runs it: roll + window at the predicted pose, insertion of the down-sized
    stacks (sensor frame) with the optimised pose (:536-577), re-filter of the valid cubes.  maps / leaves / stacks_ds:
    (corner, surface).  Returns (valid cube list, from-map clouds taken before the insertion)."""
    cen, valid, _ = window(twist_predicted, maps[0].cen)
    for m in maps:
        m.roll_to(cen)
    from_map = [m.from_map(valid) for m in maps]
    pose = Pose(twist_optimised)
    for m, stack, leaf in zip(maps, stacks_ds, leaves):
        m.add(pose.to_map(stack))
        m.filter(valid, leaf, voxel_grid)
    return valid, from_map


def voxel_face(k, leaf):
    """Smallest float32 x of the voxel with index k (floor(x * (1 / leaf)) == k, pcl::VoxelGrid's arithmetic)."""
    inv = F(1.0) / F(leaf)
    f = F(np.float64(k) * leaf)
    while np.floor(f * inv) >= k:
        f = np.nextafter(f, F(-np.inf))
    while np.floor(f * inv) < k:
        f = np.nextafter(f, F(np.inf))
    return f


def first_crossing(face, side, label, n_max=512, k_max=1024):
    """Brute force: the first (value, n) such that n copies of a float32 `value`, k <= k_max ulps from `face` on `side`
    (-1 below, +1 above), have an fp32 centroid (sequential sum, then / n) whose label differs from the value's.
    label: float32 array -> integer array (cube or voxel index).  None when there is none.  The sum and the division
    are monotone in every input, so a set of distinct values on one side cannot get closer to the face than n copies
    of its extreme value: no crossing of copies means no crossing at all (for up to n_max points)."""
    v = np.empty(k_max, F)
    x = F(face)
    for k in range(k_max):
        x = np.nextafter(x, F(side * np.inf))
        v[k] = x
    lv = label(v)
    s = np.zeros(k_max, F)
    for n in range(1, n_max + 1):
        s = (s + v).astype(F)
        moved = np.flatnonzero(label((s / F(n)).astype(F)) != lv)
        if moved.size:
            return v[moved[0]], n
    return None


def sorted_rows(a):
    """Rows in lexicographic order (multiset comparison of point clouds)."""
    a = np.asarray(a, np.float32).reshape(-1, 4)
    return a[np.lexsort(a.T[::-1])]
