"""numpy restatement of snapshots and merging of the whole-run voxel map (csrc/densemap.cuh: dense_snapshot_kernel,
dense_merge_key_kernel, dense_merge_run_kernel, dense_merge_insert_kernel; include/loam_b200.h "Whole-run voxel map
snapshots and merging").

A snapshot is the map's state itself: keys, counts, hits, misses and the fp64 sums in ascending key order.  A merge of
entries (counts, hits, misses, sums), fp64 without FMA and each operation rounded on its own, as the kernels:
  * S' = S without a pose; otherwise (Sx, Sy, Sz) rotated by rotZ, rotX, rotY (align_reference.to_map64's order) with
    math.cos / math.sin of the pose's float angles, then + count * pos per axis (float pos as double); intensity as is;
  * destination: the key of the fp32 centroid (float32)(S' / count) by the map's rule (dense_reference.voxel_keys at the
    map's leaf); not finite or outside the key range: skipped, its count added to `skipped`;
  * one destination's entries in ascending input index: P = ((0.0 + S'_1) + S'_2) + ..., counts added in uint32, hits
    and misses each added and saturated at 65535 (saturating addition of non-negative values is order-free);
  * a stored voxel gets S + P, its count + the group's, saturated evidence sums; new voxels are admitted in ascending
    key order while fewer than max_voxels are stored, the counts of the others are dropped; no hit of the merge's own.
Deliberately wrong variants (`variant=`) exist so that the tests can show their cases tell them apart:
  "fp64_centroid" (bin by the fp64 centroid), "descending" (group in descending input index), "no_saturation"
  (evidence wraps in 16 bits), "extra_hit" (one hit per merged voxel, as an insert adds) and "input_order" (admit new
  voxels in order of their first entry instead of key order).
"""
import math

import numpy as np

import dense_reference as dr
import visibility_reference as vr

SAT = vr.SAT
U32 = 0xFFFFFFFF
VARIANTS = ("fp64_centroid", "descending", "no_saturation", "extra_hit", "input_order")


def snapshot(ref):
    """The snapshot of a restated map (dense_reference / visibility_reference), as api.Ctx.dense_snapshot returns it."""
    n = ref.keys.size
    hits = getattr(ref, "hits", np.ones(n, np.int64))
    misses = getattr(ref, "misses", np.zeros(n, np.int64))
    return {"leaf": np.float32(ref.leaf), "keys": ref.keys.astype(np.uint64), "counts": ref.count.astype(np.uint32),
            "hits": np.asarray(hits).astype(np.uint16), "misses": np.asarray(misses).astype(np.uint16),
            "sums": np.array(ref.S, np.float64).reshape(-1, 4)}


def validate(snap, twist6):
    """The host checks of loam_b200_dense_merge: ValueError where the library returns LOAM_B200_ERR_ARG."""
    cnt = np.asarray(snap["counts"]).reshape(-1)
    n = cnt.size
    if (np.asarray(snap["hits"]).size != n or np.asarray(snap["misses"]).size != n
            or np.asarray(snap["sums"]).size != 4 * n):
        raise ValueError("arrays differ in length")
    if twist6 is not None and not np.all(np.isfinite(np.asarray(twist6, np.float32))):
        raise ValueError("pose not finite")
    if (cnt == 0).any():
        raise ValueError("count 0")
    if (np.asarray(snap["hits"]) == 0).any():
        raise ValueError("hits 0")
    if not np.all(np.isfinite(np.asarray(snap["sums"], np.float64))):
        raise ValueError("sum not finite")


def transform_sums(counts, S, twist6):
    """S' of the entries (N x 4 float64)."""
    S = np.array(S, np.float64).reshape(-1, 4)
    if twist6 is None:
        return S
    t = np.asarray(twist6, np.float32)
    cx, sx = math.cos(float(t[0])), math.sin(float(t[0]))
    cy, sy = math.cos(float(t[1])), math.sin(float(t[1]))
    cz, sz = math.cos(float(t[2])), math.sin(float(t[2]))
    x, y, z = S[:, 0], S[:, 1], S[:, 2]
    x1 = cz * x - sz * y
    y1 = sz * x + cz * y
    y2 = cx * y1 - sx * z
    z2 = sx * y1 + cx * z
    c = np.asarray(counts).astype(np.float64)
    out = S.copy()
    out[:, 0] = (cy * x1 + sy * z2) + c * float(t[3])
    out[:, 1] = y2 + c * float(t[4])
    out[:, 2] = (cy * z2 - sy * x1) + c * float(t[5])
    return out


def destination_keys(counts, S2, leaf, fp64_centroid=False):
    """Key of each entry's centroid at `leaf` (EMPTY: skipped)."""
    c = np.asarray(counts).astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        c64 = S2[:, :3] / c[:, None]
        if not fp64_centroid:
            c32 = c64.astype(np.float32)
            return dr.voxel_keys(np.concatenate([c32, np.zeros((c32.shape[0], 1), np.float32)], axis=1), leaf)
        inv = float(np.float32(1.0) / np.float32(leaf))
        f = np.floor(c64 * inv)
        ok = np.all(np.isfinite(f) & (f >= -dr.HALF) & (f < dr.HALF), axis=1)
    v = np.zeros((c64.shape[0], 3), np.uint64)
    v[ok] = (f[ok].astype(np.int64) + dr.HALF).astype(np.uint64)
    k = (v[:, 2] << np.uint64(42)) | (v[:, 1] << np.uint64(21)) | v[:, 0]
    k[~ok] = dr.EMPTY
    return k


class MergeMapRef(vr.VisibilityMapRef):
    """VisibilityMapRef + snapshot() and merge()."""

    def snapshot(self):
        return snapshot(self)

    def state(self):
        """(keys, counts, sum bits, hits, misses): what two maps must share to be the same map."""
        return (self.keys.copy(), self.count.astype(np.uint32), np.array(self.S, np.float64).view(np.uint64).copy(),
                self.hits.astype(np.uint16), self.misses.astype(np.uint16))

    def merge(self, snap, twist6=None, variant=None):
        """Merge the snapshot's entries -> {"stored", "new", "skipped", "dropped"}: where the merged counts went."""
        assert variant is None or variant in VARIANTS
        validate(snap, twist6)
        cnt = np.asarray(snap["counts"], np.uint32).reshape(-1).astype(np.int64)
        h = np.asarray(snap["hits"], np.uint16).reshape(-1).astype(np.int64)
        m = np.asarray(snap["misses"], np.uint16).reshape(-1).astype(np.int64)
        out = {"stored": 0, "new": 0, "skipped": 0, "dropped": 0}
        if cnt.size == 0:
            return out
        S2 = transform_sums(cnt, snap["sums"], twist6)
        keys = destination_keys(cnt, S2, self.leaf, variant == "fp64_centroid")
        skip = keys == dr.EMPTY
        out["skipped"] = int(cnt[skip].sum())
        self.skipped += out["skipped"]
        idx = np.nonzero(~skip)[0]
        if idx.size == 0:
            return out
        if variant == "descending":
            order = idx[np.lexsort((-idx, keys[idx]))]
        else:
            order = idx[np.argsort(keys[idx], kind="stable")]
        uk, start, size = np.unique(keys[order], return_index=True, return_counts=True)
        P = np.zeros((uk.size, 4), np.float64)
        for j in range(int(size.max())):
            sel = size > j
            P[sel] = P[sel] + S2[order[start[sel] + j]]
        gc = np.add.reduceat(cnt[order], start) & U32
        gh = np.add.reduceat(h[order], start)
        gm = np.add.reduceat(m[order], start)
        first = np.minimum.reduceat(order, start)

        def sat(e):
            return e & 0xFFFF if variant == "no_saturation" else np.minimum(e, SAT)

        gh, gm = sat(gh), sat(gm)
        if variant == "extra_hit":
            gh = sat(gh + 1)
        pos = np.searchsorted(self.keys, uk)
        found = pos < self.keys.size
        found[found] = self.keys[pos[found]] == uk[found]
        at = pos[found]
        self.S[at] = self.S[at] + P[found]
        self.count[at] = (self.count[at] + gc[found]) & U32
        self.hits[at] = sat(self.hits[at] + gh[found])
        self.misses[at] = sat(self.misses[at] + gm[found])
        out["stored"] = int(gc[found].sum())
        new = np.nonzero(~found)[0]  # ascending key order
        if variant == "input_order":
            new = new[np.argsort(first[new], kind="stable")]
        room = max(self.max_voxels - self.keys.size, 0)
        adm, rej = np.sort(new[:room]), new[room:]
        out["new"] = int(gc[adm].sum())
        out["dropped"] = int(gc[rej].sum())
        self.dropped += out["dropped"]
        k = np.concatenate([self.keys, uk[adm]])
        o = np.argsort(k, kind="stable")
        self.keys = k[o]
        self.count = np.concatenate([self.count, gc[adm]])[o]
        self.S = np.concatenate([self.S, P[adm]])[o]
        self.hits = np.concatenate([self.hits, gh[adm]])[o]
        self.misses = np.concatenate([self.misses, gm[adm]])[o]
        return out


def entries(rows):
    """A snapshot dict from rows (count, hits, misses, sx, sy, sz, si)."""
    r = np.asarray(rows, np.float64).reshape(-1, 7)
    return {"leaf": None, "keys": np.zeros(r.shape[0], np.uint64), "counts": r[:, 0].astype(np.uint32),
            "hits": r[:, 1].astype(np.uint16), "misses": r[:, 2].astype(np.uint16), "sums": r[:, 3:].copy()}


def concat(*snaps):
    return {f: np.concatenate([s[f] for s in snaps]) for f in ("keys", "counts", "hits", "misses", "sums")} | \
        {"leaf": None}


HAND_LEAF = 0.5  # 1 / leaf is exact; the faces below are exact in fp32


def hand_cases():
    """-> {name: (max_voxels, the map's initial entries or None, entries to merge, twist6 or None)}.  Every case is
    merged into a map of HAND_LEAF that first receives its initial entries (merged with no pose)."""
    f32 = np.float32
    up = float(np.nextafter(f32(1.5), f32(np.inf)))
    down = float(np.nextafter(f32(1.5), f32(-np.inf)))
    a, b, c = (4, 1, 0, 1.0, 0.4, 0.4, 1.0), (1, 1, 0, 1e-16, 0.1, 0.1, 2.0), (1, 1, 0, 1e-16, 0.1, 0.1, 3.0)
    cases = {
        # three entries of voxel (0, 0, 0) whose fp64 sum depends on the order: (1 + 1e-16) + 1e-16 = 1 but
        # (1e-16 + 1e-16) + 1 > 1; and two entries of one voxel in both orders
        "one_voxel_order_abc": (2**31 - 1, None, entries([a, b, c]), None),
        "one_voxel_order_cba": (2**31 - 1, None, entries([c, b, a]), None),
        "two_entries_ab": (2**31 - 1, None, entries([a, b]), None),
        "two_entries_ba": (2**31 - 1, None, entries([b, a]), None),
        # the face x = 1.5 (voxel 3 of leaf 0.5) after a translation of 0.25: on it, one fp32 ulp either side, and an
        # fp64 centroid just below the face that rounds onto it in fp32
        "face": (2**31 - 1, None, entries([(1, 1, 0, 1.25, 0.2, 0.2, 1.0), (1, 2, 0, up - 0.25, 0.2, 0.2, 1.0),
                                           (1, 3, 0, down - 0.25, 0.2, 0.2, 1.0),
                                           (2, 4, 0, 2.5 - 2e-12, 0.4, 0.4, 1.0),
                                           (3, 5, 0, 3 * 1.25 - 1e-12, 0.6, 0.6, 1.0)]),
                 (0.0, 0.0, 0.0, 0.25, 0.0, 0.0)),
        # evidence near 65535: in one group, and added to a stored voxel
        "saturation": (2**31 - 1, entries([(1, 65530, 65000, 0.1, 0.1, 0.1, 1.0)]),
                       entries([(1, 3, 300, 0.2, 0.2, 0.2, 1.0), (1, 4, 400, 0.1, 0.2, 0.1, 1.0),
                                (1, 65000, 65535, 5.1, 0.1, 0.1, 1.0), (1, 600, 1, 5.2, 0.2, 0.2, 1.0),
                                (1, 65534, 2, 9.1, 0.1, 0.1, 1.0)]), None),
        # a translation that moves some entries past the key range (2^20 voxels of 0.5 m = 524288 m)
        "key_range": (2**31 - 1, None, entries([(1, 1, 0, 10.0, 0.1, 0.1, 1.0), (1, 1, 0, -30.0, 0.1, 0.1, 1.0),
                                                (2, 1, 0, -2.0, 0.2, 0.2, 1.0)]),
                      (0.0, 0.0, 0.0, 524280.0, 0.0, 0.0)),
        # cap 5 with 3 stored: of four new voxels (given in descending key order) the two lowest keys are admitted
        "cap": (5, entries([(1, 1, 0, 0.1, 0.1, 0.1, 1.0), (1, 1, 0, 1.1, 0.1, 0.1, 1.0), (1, 1, 0, 2.1, 0.1, 0.1, 1.0)]),
                entries([(1, 1, 0, 9.1, 0.1, 0.1, 1.0), (2, 2, 1, 14.2, 0.2, 0.2, 2.0), (1, 1, 0, 0.2, 0.2, 0.2, 1.0),
                         (1, 1, 0, 5.1, 0.1, 0.1, 1.0), (1, 1, 0, 3.1, 0.1, 0.1, 1.0)]), None),
        # into voxels already stored, under a rotation about y
        "stored": (2**31 - 1, entries([(2, 3, 1, 0.6, 0.2, 0.4, 3.0), (1, 1, 0, 2.3, 0.1, -0.7, 1.0)]),
                   entries([(1, 1, 0, -0.2, 0.1, 0.3, 1.0), (1, 2, 2, -0.7, 0.1, -2.3, 4.0)]),
                   (0.0, np.float32(math.pi / 2), 0.0, 0.0, 0.0, 0.0)),
    }
    return cases


def run_case(case, variant=None):
    """The restated map after a hand-made case -> MergeMapRef."""
    max_voxels, initial, merged, twist = case
    ref = MergeMapRef(HAND_LEAF, max_voxels)
    if initial is not None:
        ref.merge(initial)
    ref.merge(merged, twist, variant)
    return ref
