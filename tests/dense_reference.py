"""numpy restatement of the whole-run voxel map (csrc/densemap.cuh; include/loam_b200.h "Whole-run voxel map").

Every step is written so that its floating-point operations are the ones the GPU performs, in the same order:
  * voxel of a point: floorf(c * (1.0f / leaf)) per axis in fp32, range [-2^20, 2^20) checked in float;
  * key = (v_z + 2^20) << 42 | (v_y + 2^20) << 21 | (v_x + 2^20);
  * per sweep and voxel, the points are summed in fp64 one after the other in ascending cloud index, starting from 0.0
    (numpy's add.reduce / reduceat sum pairwise, which is a different order: the sums are vectorised across voxels by
    looping over the position inside a voxel instead, and long runs use add.accumulate, which is sequential);
  * the stored sum of a voxel is S = ((P1 + P2) + P3) + ... over the sweeps in order;
  * export: (float32)(S / count) per field, voxels in ascending key order;
  * a sweep's new voxels are admitted in ascending key order while fewer than max_voxels voxels are stored; the points of
    the others are dropped.
"""
import numpy as np

HALF = 1 << 20
LIM = np.float32(HALF)
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)
LONG_RUN = 256  # runs longer than this are summed one by one with add.accumulate


def voxel_keys(pts, leaf):
    """uint64 key per point; EMPTY for a skipped point (not finite, or a voxel outside the key range)."""
    p = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 4)
    inv = np.float32(1.0) / np.float32(leaf)
    with np.errstate(invalid="ignore", over="ignore"):
        f = np.floor(p[:, :3] * inv)
        ok = np.all((f >= -LIM) & (f < LIM), axis=1)
    v = np.zeros((p.shape[0], 3), np.uint64)
    v[ok] = (f[ok].astype(np.int64) + HALF).astype(np.uint64)
    k = (v[:, 2] << np.uint64(42)) | (v[:, 1] << np.uint64(21)) | v[:, 0]
    k[~ok] = EMPTY
    return k


def key_voxel(k):
    """(v_x, v_y, v_z) of keys."""
    k = np.asarray(k, np.uint64)
    m = np.uint64((1 << 21) - 1)
    return np.stack([(k & m).astype(np.int64) - HALF, ((k >> np.uint64(21)) & m).astype(np.int64) - HALF,
                     (k >> np.uint64(42)).astype(np.int64) - HALF], axis=1)


def sweep_partials(pts, leaf):
    """One cloud -> (sorted unique keys, counts, fp64 partial sums P (n_voxels x 4), skipped points)."""
    p = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 4)
    k = voxel_keys(p, leaf)
    ok = k != EMPTY
    skipped = int((~ok).sum())
    idx = np.nonzero(ok)[0]
    order = idx[np.argsort(k[idx], kind="stable")]  # stable: ascending cloud index inside a voxel
    sk = k[order]
    if sk.size == 0:
        return np.zeros(0, np.uint64), np.zeros(0, np.int64), np.zeros((0, 4), np.float64), skipped
    keys, start, counts = np.unique(sk, return_index=True, return_counts=True)
    vals = p[order].astype(np.float64)
    P = np.zeros((keys.size, 4), np.float64)
    short = counts <= LONG_RUN
    for j in range(int(counts[short].max()) if short.any() else 0):
        sel = short & (counts > j)
        P[sel] = P[sel] + vals[start[sel] + j]
    for r in np.nonzero(~short)[0]:
        run = np.concatenate([np.zeros((1, 4)), vals[start[r]:start[r] + counts[r]]])
        P[r] = np.add.accumulate(run, axis=0)[-1]
    return keys, counts.astype(np.int64), P, skipped


class DenseMapRef:
    def __init__(self, leaf, max_voxels=2**31 - 1):
        self.leaf = np.float32(leaf)
        self.max_voxels = int(max_voxels)
        self.keys = np.zeros(0, np.uint64)
        self.count = np.zeros(0, np.int64)
        self.S = np.zeros((0, 4), np.float64)
        self.skipped = 0
        self.dropped = 0

    def insert(self, pts):
        keys, counts, P, skipped = sweep_partials(pts, self.leaf)
        self.skipped += skipped
        pos = np.searchsorted(self.keys, keys)
        found = pos < self.keys.size
        found[found] = self.keys[pos[found]] == keys[found]
        at = pos[found]
        self.S[at] = self.S[at] + P[found]  # one fp64 add per field: S_new = S_old + P
        self.count[at] += counts[found]
        new = np.nonzero(~found)[0]  # ascending key order
        room = max(self.max_voxels - self.keys.size, 0)
        adm, rej = new[:room], new[room:]
        self.dropped += int(counts[rej].sum())
        k = np.concatenate([self.keys, keys[adm]])
        o = np.argsort(k, kind="stable")
        self.keys = k[o]
        self.count = np.concatenate([self.count, counts[adm]])[o]
        self.S = np.concatenate([self.S, P[adm]])[o]

    def stats(self):
        return {"voxels": int(self.keys.size), "skipped": self.skipped, "dropped": self.dropped}

    def export(self):
        """(centroids N x 4 float32, counts N uint32) in ascending key order."""
        with np.errstate(invalid="ignore"):
            c = (self.S / self.count[:, None].astype(np.float64)).astype(np.float32)
        return c.reshape(-1, 4), self.count.astype(np.uint32)


def key_edge_cloud(leaf):
    """Hand-made points on the edges of the key: voxel faces and 1 ulp below, -0.0, negative coordinates, the key range
    limits +-2^20 and one voxel beyond, NaN and inf.  Intensities are distinct so that averaging shows up."""
    leaf = np.float32(leaf)
    inv = np.float32(1.0) / leaf
    rows = []

    def add(x, y, z):
        rows.append((np.float32(x), np.float32(y), np.float32(z), np.float32(len(rows) % 7)))

    for m in (0, 1, 3, -1, -3, 17, -17):
        # the smallest float whose voxel is m on x (a voxel face as the key computes it) and the float just below it
        face = np.float32(m) * leaf
        while np.floor(face * inv) > m:
            face = np.nextafter(face, np.float32(-np.inf))
        while np.floor(face * inv) < m:
            face = np.nextafter(face, np.float32(np.inf))
        while np.floor(np.nextafter(face, np.float32(-np.inf)) * inv) >= m:
            face = np.nextafter(face, np.float32(-np.inf))
        below = np.nextafter(face, np.float32(-np.inf))
        for x in (face, below):
            add(x, 0.5 * leaf, -0.5 * leaf)
            add(-0.25 * leaf, x, 2.5 * leaf)
            add(1.5 * leaf, -2.5 * leaf, x)
    add(-0.0, -0.0, -0.0)
    add(0.0, -0.0, 0.0)
    add(-1e-30, 1e-30, -1e-30)
    for s in (1, -1):
        # the outermost voxels of the range, the first voxels beyond it, and points far outside
        inside = np.float32(s * (HALF - 1)) * leaf if s > 0 else np.float32(-HALF) * leaf
        beyond = np.float32(s * HALF) * leaf if s > 0 else np.nextafter(np.float32(-HALF) * leaf, np.float32(-np.inf))
        for c in (inside, beyond, np.float32(s * 3e38)):
            add(c, 0.0, 0.0)
            add(0.0, c, 0.0)
            add(0.0, 0.0, c)
    for bad in (np.nan, np.inf, -np.inf):
        add(bad, 0.0, 0.0)
        add(0.0, bad, 0.0)
        add(0.0, 0.0, bad)
    return np.array(rows, np.float32)
