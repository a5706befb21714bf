"""numpy restatement of the visibility pass of the whole-run voxel map (csrc/densemap.cuh: dense_pixel,
dense_range_image_kernel, dense_visibility_kernel; include/loam_b200.h "loam_b200_dense_visibility").

Everything is double, and every product and sum is written out in the order the kernels use (the library is built
without FMA contraction):
  * map frame -> sensor frame: d = c - pos, then rotY(-rot_y), rotX(-rot_x), rotZ(-rot_z) with the expressions of
    math_utils.h (pointAssociateTobeMapped, BasicLaserMapping.cpp:223-231); cos / sin of the negated float angles in
    double from math.cos / math.sin (the libm the library's host code calls; numpy's vectorised cos may differ);
  * r = sqrt((x*x + y*y) + z*z), elevation atan2(y, sqrt(x*x + z*z)), azimuth atan2(x, z);
  * row = clamp(floor((deg(e) + 90) / v_res), 0, rows - 1), col = floor((deg(a) + 180) / h_res) mod cols, with
    deg(u) = u * (180 / pi);
  * range image: per pixel the minimum (float32) r over the sweep's finite points with r > 0;
  * a stored voxel (centroid sum / count in double) gets a miss when its pixel holds a finite value v and
    (double) v > r + margin; every voxel that receives points in an insert gets a hit; both saturate at 65535.
atan2 of the GPU may differ from this one in the last ulp, so observe() also reports the voxels within EDGE of a pixel
edge or of the miss threshold, whose miss may legitimately differ.
"""
import math

import numpy as np

import dense_reference as dr

RAD2DEG = 180.0 / math.pi
SAT = 65535
EDGE = 1e-9


def image_shape(h_res, v_res):
    return int(math.ceil(180.0 / v_res)), int(math.ceil(360.0 / h_res))


def sensor_frame(c, twist6):
    """(N, 3) float64 map-frame positions -> x, y, z in the sensor frame of twist6 = (rot_x, rot_y, rot_z, x, y, z)."""
    t6 = np.asarray(twist6, np.float32)
    c = np.asarray(c, np.float64).reshape(-1, 3)
    x = c[:, 0] - float(t6[3])
    y = c[:, 1] - float(t6[4])
    z = c[:, 2] - float(t6[5])
    cy, sy = math.cos(-float(t6[1])), math.sin(-float(t6[1]))
    cx, sx = math.cos(-float(t6[0])), math.sin(-float(t6[0]))
    cz, sz = math.cos(-float(t6[2])), math.sin(-float(t6[2]))
    t = x
    x = cy * t + sy * z
    z = cy * z - sy * t
    t = y
    y = cx * t - sx * z
    z = sx * t + cx * z
    t = x
    x = cz * t - sz * y
    y = sz * t + cz * y
    return x, y, z


def _coords(c, twist6, h_res, v_res):
    """-> r, unclamped row and column coordinates ur, uc (pixel = floor of each), row, col per position."""
    rows, cols = image_shape(h_res, v_res)
    x, y, z = sensor_frame(c, twist6)
    r = np.sqrt((x * x + y * y) + z * z)
    e = np.arctan2(y, np.sqrt(x * x + z * z))
    a = np.arctan2(x, z)
    ur = (e * RAD2DEG + 90.0) / v_res
    uc = (a * RAD2DEG + 180.0) / h_res
    row = np.clip(np.floor(ur), 0, rows - 1).astype(np.int64)
    col = np.floor(uc).astype(np.int64) % cols
    return r, ur, uc, row, col


def pixels(c, twist6, h_res, v_res):
    """-> (r, pixel index, near_edge) per position; near_edge: within EDGE of a row or column boundary."""
    cols = image_shape(h_res, v_res)[1]
    r, ur, uc, row, col = _coords(c, twist6, h_res, v_res)
    near = (np.abs(ur - np.round(ur)) < EDGE) | (np.abs(uc - np.round(uc)) < EDGE)
    return r, row * cols + col, near


def range_image(pts, twist6, h_res, v_res):
    """-> (image float32 rows*cols, +inf where no return; pixels an edge point may fall into instead)."""
    rows, cols = image_shape(h_res, v_res)
    p = np.asarray(pts, np.float32).reshape(-1, 4)
    ok = np.all(np.isfinite(p[:, :3]), axis=1)
    q = p[ok, :3].astype(np.float64)
    r, ur, uc, row, col = _coords(q, twist6, h_res, v_res)
    img = np.full(rows * cols, np.inf, np.float32)
    pos = r > 0.0
    np.minimum.at(img, (row * cols + col)[pos], r[pos].astype(np.float32))
    # a point within EDGE of a boundary may land on the other side of it on the GPU: its own pixel and the one across
    # (row, column or both) are uncertain
    fr, fc = ur - np.floor(ur), uc - np.floor(uc)
    dr_ = np.where(fr < EDGE, -1, np.where(fr > 1.0 - EDGE, 1, 0))
    dc = np.where(fc < EDGE, -1, np.where(fc > 1.0 - EDGE, 1, 0))
    edge = pos & ((dr_ != 0) | (dc != 0))
    row, col, dr_, dc = row[edge], col[edge], dr_[edge], dc[edge]
    unsure = np.zeros(rows * cols, bool)
    for sr, sc in ((0, 0), (1, 0), (0, 1), (1, 1)):
        unsure[np.clip(row + sr * dr_, 0, rows - 1) * cols + (col + sc * dc) % cols] = True
    return img, unsure


def miss_mask(cent, img, unsure, twist6, h_res, v_res, margin):
    """-> (miss, uncertain) per centroid (N x 3 float64)."""
    r, pix, near = pixels(cent, twist6, h_res, v_res)
    v = img[pix].astype(np.float64)
    thr = r + margin
    fin = np.isfinite(v)
    miss = fin & (v > thr)
    uncertain = near | unsure[pix] | (fin & (np.abs(v - thr) < EDGE))
    return miss, uncertain


class VisibilityMapRef(dr.DenseMapRef):
    """DenseMapRef + per-voxel hits and misses (aligned with self.keys) and the visibility pass."""

    def __init__(self, leaf, max_voxels=2**31 - 1, h_res=0.0, v_res=1.0, margin=0.0):
        super().__init__(leaf, max_voxels)
        self.hits = np.zeros(0, np.int64)
        self.misses = np.zeros(0, np.int64)
        self.set_visibility(h_res, v_res, margin)
        self.uncertain = set()  # keys whose miss count may differ from the GPU's by atan2's last ulp

    def set_visibility(self, h_res, v_res, margin):
        self.h_res, self.v_res, self.margin = float(h_res), float(v_res), float(margin)

    def centroids(self):
        return self.S[:, :3] / self.count[:, None].astype(np.float64)

    def observe(self, pts, twist6):
        """The pass over one map-frame cloud seen from twist6 (before that cloud's insert)."""
        if self.h_res == 0.0 or self.keys.size == 0 or np.asarray(pts).size == 0:
            return
        img, unsure = range_image(pts, twist6, self.h_res, self.v_res)
        miss, unc = miss_mask(self.centroids(), img, unsure, twist6, self.h_res, self.v_res, self.margin)
        self.misses = np.minimum(self.misses + miss, SAT)
        self.uncertain.update(int(k) for k in self.keys[unc])

    def insert(self, pts):
        old_keys, old_h, old_m = self.keys, self.hits, self.misses
        super().insert(pts)
        h = np.zeros(self.keys.size, np.int64)
        m = np.zeros(self.keys.size, np.int64)
        at = np.searchsorted(self.keys, old_keys)
        h[at], m[at] = old_h, old_m
        k = np.unique(dr.voxel_keys(pts, self.leaf))
        k = k[k != dr.EMPTY]
        pos = np.searchsorted(self.keys, k)
        ok = pos < self.keys.size
        ok[ok] = self.keys[pos[ok]] == k[ok]
        h[pos[ok]] = np.minimum(h[pos[ok]] + 1, SAT)
        self.hits, self.misses = h, m

    def sweep(self, pts, twist6):
        """What the mapping stage does at the end of a sweep: observe, then insert."""
        self.observe(pts, twist6)
        self.insert(pts)

    def keep_mask(self, max_miss_ratio):
        return self.misses.astype(np.float64) <= float(max_miss_ratio) * self.hits.astype(np.float64)

    def export_filtered(self, max_miss_ratio=math.inf):
        """(centroids, counts, hits, misses) of the voxels with misses <= max_miss_ratio * hits, ascending key order."""
        c, n = self.export()
        keep = self.keep_mask(max_miss_ratio)
        return c[keep], n[keep], self.hits[keep].astype(np.uint16), self.misses[keep].astype(np.uint16)


# ---- a moving box in the synthetic street scene, registered with the ground-truth poses
BOX_SIZE = (4.5, 1.6, 1.8)  # length (along its motion, x), height, width (z)


def box_at(k, speed=10.0, z_centre=7.0, x0=-14.0, scan_period=0.1):
    """Box of sweep k: driving along +x across the street in front of the sensor (bottom on the ground)."""
    from loam_velodyne_b200 import synth
    cx = x0 + speed * scan_period * k
    L, H, W = BOX_SIZE
    return np.array([cx - L / 2, cx + L / 2, -synth.SENSOR_HEIGHT, -synth.SENSOR_HEIGHT + H,
                     z_centre - W / 2, z_centre + W / 2])


def moving_box_run(scene, lidar, n_sweeps, v=(0.0, 0.0, 1.0), yaw_rate=math.radians(5.0), scan_period=0.1):
    """-> list of (registered cloud N x 4 float32 in the map frame, twist6 of the sweep, box-point mask).  Each point
    is registered with the pose at its own firing time (ground truth, no de-skew error); the sweep's pose is the one at
    mid-sweep."""
    import dataclasses

    from loam_velodyne_b200 import synth
    out = []
    vv = np.asarray(v, np.float64)
    for k in range(n_sweeps):
        box = box_at(k, scan_period=scan_period)
        sc = dataclasses.replace(scene, boxes=np.vstack([scene.boxes, box[None, :]]))
        pts, _ = synth.make_sweep(sc, lidar, k, scan_period=scan_period, v=v, yaw_rate=yaw_rate)
        A = lidar.n_az
        assert pts.shape[0] == lidar.n_rings * A  # every ray returns: azimuth index = i mod n_az
        frac = (np.arange(pts.shape[0]) % A).astype(np.float64) / A
        t0 = k * scan_period
        pos = np.empty((A, 3))
        yaw = np.empty(A)
        for a in range(A):
            pos[a], yaw[a] = synth.pose_at(t0 + a / A * scan_period, vv, yaw_rate)
        ia = np.arange(pts.shape[0]) % A
        c, s = np.cos(yaw[ia]), np.sin(yaw[ia])
        p = pts[:, :3].astype(np.float64)
        w = np.stack([c * p[:, 0] + s * p[:, 2] + pos[ia, 0], p[:, 1] + pos[ia, 1],
                      -s * p[:, 0] + c * p[:, 2] + pos[ia, 2]], axis=1)
        reg = np.concatenate([w.astype(np.float32), pts[:, 3:4]], axis=1)
        pm, ym = synth.pose_at(t0 + 0.5 * scan_period, vv, yaw_rate)
        twist = np.array([0.0, ym, 0.0, pm[0], pm[1], pm[2]], np.float32)
        e = 0.05
        in_box = ((w[:, 0] > box[0] - e) & (w[:, 0] < box[1] + e) & (w[:, 1] > box[2] - e) & (w[:, 1] < box[3] + e) &
                  (w[:, 2] > box[4] - e) & (w[:, 2] < box[5] + e))
        out.append((np.ascontiguousarray(reg), twist, in_box))
    return out


def trail_and_static(run, leaf, settle=6):
    """Voxel keys of the trail (only box points, the last of them at least `settle` sweeps before the end: the box has
    left them) and of the static map (no box point ever)."""
    box_last = {}
    static = set()
    for k, (pts, _, in_box) in enumerate(run):
        kb = np.unique(dr.voxel_keys(pts[in_box], leaf))
        ks = np.unique(dr.voxel_keys(pts[~in_box], leaf))
        for x in kb.tolist():
            box_last[x] = k
        static.update(ks.tolist())
    trail = {x for x, k in box_last.items() if x not in static and k <= len(run) - 1 - settle}
    static -= set(box_last)
    return trail, static


def removal_rates(ref, trail, static, max_miss_ratio):
    keep = ref.keep_mask(max_miss_ratio)
    keys = ref.keys.tolist()
    kept = {k for k, f in zip(keys, keep.tolist()) if f}
    return (1.0 - len(trail & kept) / max(len(trail), 1), len(static & kept) / max(len(static), 1))
