"""numpy restatement of the relocalisation against the whole-run voxel map (csrc/stages.inc: loam_b200_reloc_grid,
loam_b200_dense_relocalize; include/loam_b200.h "Relocalisation against the whole-run voxel map").

The grid is restated in float32 operation by operation; the rules of the pipeline (keep, rank, dedup) are plain
Python over score tables.  Scoring and refinement are compositions of align_reference.iterate / align, or of the
library's dense_score / dense_align_batch when a test replays the pipeline on the GPU.
"""
import math

import numpy as np

import align_reference as ar
from loam_velodyne_b200.api import sincos_f32

F = np.float32
MIN_SELECTED = 50  # below this an alignment cannot take a step, so the hypothesis is never kept


def grid(prior6, yaw_step_deg, yaw_steps, xz_step, xz_steps):
    """-> (K x 6 float32 twists, K x 3 sin, K x 3 cos): j (yaw) outer, then iz, then ix, each ascending."""
    p = np.asarray(prior6, np.float32)
    step, xs = F(yaw_step_deg), F(xz_step)
    tw = []
    for j in range(-yaw_steps, yaw_steps + 1):
        ry = F(p[1] + F(float(j) * float(step) * math.pi / 180.0))
        for iz in range(-xz_steps, xz_steps + 1):
            for ix in range(-xz_steps, xz_steps + 1):
                tw.append([p[0], ry, p[2], F(p[3] + F(F(ix) * xs)), p[4], F(p[5] + F(F(iz) * xs))])
    tw = np.array(tw, np.float32).reshape(-1, 6)
    sc = np.array([[sincos_f32(a) for a in t[:3]] for t in tw], np.float32).reshape(-1, 3, 2)
    return tw, sc[:, :, 0].copy(), sc[:, :, 1].copy()


def keep_rule(n_selected, keep, larger_index_first=False, keep_below_min=False):
    """Indices kept: n_selected >= 50, by n_selected descending then index ascending, the first `keep`.  The keywords
    are deliberately wrong variants of the sensitivity tests."""
    idx = [h for h in range(len(n_selected)) if keep_below_min or n_selected[h] >= MIN_SELECTED]
    idx.sort(key=lambda h: (-int(n_selected[h]), -h if larger_index_first else h))
    return idx[:keep]


def rms_of(n_selected, sum_sq):
    return F(math.sqrt(float(sum_sq) / float(n_selected))) if n_selected > 0 else F(0.0)


def rank_rule(selected, rms, rms_descending=False):
    """Positions 0..K-1 ranked by selected descending, then rms ascending, then position."""
    return sorted(range(len(selected)),
                  key=lambda j: (-int(selected[j]), -float(rms[j]) if rms_descending else float(rms[j]), j))


def dedup_rule(twists, ranked, dedup_m, dedup_deg, cap, le=False):
    """The survivors of `ranked` (positions into twists): a candidate within dedup_m in translation AND dedup_deg in
    rotation of a better-ranked survivor is dropped; at most cap.  le=True: <= at the thresholds (wrong variant)."""
    out = []
    for j in ranked:
        dup = False
        for s in out:
            dm, ddeg = ar.twist_error(twists[j], twists[s])
            if (dm <= dedup_m and ddeg <= dedup_deg) if le else (dm < dedup_m and ddeg < dedup_deg):
                dup = True
                break
        if not dup:
            out.append(j)
            if len(out) == cap:
                break
    return out


def relocalize(score, align, hyps, prm, cap):
    """The pipeline of loam_b200_dense_relocalize.  score(twists, radius) -> (n_selected, sum_pd2_sq);
    align(twists, radius, max_iterations) -> (twists K x 6, infos); prm: api.RelocParams.  -> candidate dicts as
    api.Ctx.dense_relocalize returns them."""
    hyps = np.asarray(hyps, np.float32).reshape(-1, 6)
    sel, _ = score(hyps, prm.score_radius)
    kept = keep_rule(sel, prm.keep)
    if not kept:
        return []
    ct, cinfo = align(hyps[kept], prm.coarse_radius, prm.max_iterations)
    ft, finfo = align(ct, prm.fine_radius, prm.max_iterations)
    fsel, fss = score(ft, prm.fine_radius)
    rms = [rms_of(int(fsel[j]), fss[j]) for j in range(len(kept))]
    ranked = rank_rule(fsel, rms)
    out = []
    for j in dedup_rule(ft, ranked, float(F(prm.dedup_m)), float(F(prm.dedup_deg)), cap):
        out.append({"hypothesis": kept[j], "score_selected": int(sel[kept[j]]),
                    "coarse": (np.asarray(ct[j], np.float32), cinfo[j]), "fine": (np.asarray(ft[j], np.float32), finfo[j]),
                    "selected": int(fsel[j]), "rms": rms[j]})
    return out


def reference_score(target, pts):
    """score() of relocalize() from the iteration restatement."""
    def score(twists, radius):
        sel, ss = [], []
        for t in twists:
            _, _, n_sel, s = ar.normal_eq(ar.iterate(target, pts, t, radius)[0])
            sel.append(n_sel)
            ss.append(s)
        return np.array(sel, np.int32), np.array(ss, np.float32)
    return score


def reference_align(target, pts, drv=None):
    """align() of relocalize() from the loop restatement."""
    def align(twists, radius, max_iterations):
        outs = [ar.align(target, pts, t, radius, max_iterations, drv=drv) for t in twists]
        return np.array([o[0] for o in outs], np.float32).reshape(-1, 6), [o[1] for o in outs]
    return align
