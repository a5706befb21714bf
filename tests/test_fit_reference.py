"""Pins tests/fit_reference.py (the per-correspondence line and plane fits) to the checker bit for bit, checks that its
catalogue reaches the degenerate branches it names, and compares the fp32 arithmetic with a float64 answer."""
import math

import numpy as np
import pytest

import fit_reference as fr
import map_reference as mr

ZERO = np.zeros(6, np.float32)
YAW = np.array([0.01, 1.3, -0.02, 3.0, 0.2, 5.0], np.float32)  # a rotated pose (test_map_stage.py's "yaw")
TWIST = np.array([1.5e-3, -8e-3, 6e-4, -0.03, 0.01, -0.2], np.float32)
# float64 bars, calibrated on the catalogue and the VLP-16 sweep (7 830 fits, worst 36 eps32 * cond):
# |fp32 - float64| <= K * eps32 * cond * max(1, |c|) per coefficient, cond as fit_reference.map_*_fit64 define it
K_CORNER = 64.0
K_SURF = 64.0


@pytest.fixture(scope="module")
def catalogue(oracle):
    return fr.cases(0, oracle)


def to_sensor(twist, q_map):
    """Sensor-frame points whose pointAssociateToMap lands on q_map (float64 inverse, rounded once)."""
    p = mr.Pose(twist)
    sx, sy, sz = (float(v) for v in p.s)
    cx, cy, cz = (float(v) for v in p.c)
    q = np.asarray(q_map, np.float64)[:, :3] - np.asarray(p.pos, np.float64)
    x3, y2, z3 = q[:, 0], q[:, 1], q[:, 2]
    x1 = cy * x3 - sy * z3   # undo rot y
    z2 = sy * x3 + cy * z3
    y1 = cx * y2 + sx * z2   # undo rot x
    z = -sx * y2 + cx * z2
    x = cz * x1 + sz * y1    # undo rot z
    y = -sz * x1 + cz * y1
    out = np.zeros((q.shape[0], 4), np.float32)
    out[:, 0], out[:, 1], out[:, 2] = x, y, z
    return out


def batches(cs):
    out = {}
    for c in cs:
        out.setdefault(c.batch, []).append(c)
    return out


def batch_clouds(group, twist):
    """(corner map, surface map, corner queries, surface queries) of one batch; queries in the sensor frame."""
    cm = [c for c in group if c.kind == "corner"]
    sm = [c for c in group if c.kind == "surf"]

    def cloud(cs):
        if not cs:
            return np.zeros((0, 4), np.float32)
        p = np.concatenate([c.pts for c in cs])
        return np.concatenate([p, np.full((p.shape[0], 1), 1.0, np.float32)], axis=1)

    def qs(cs):
        if not cs:
            return np.zeros((0, 4), np.float32)
        q = np.stack([c.q for c in cs])
        return to_sensor(twist, q) if np.any(twist) else np.concatenate([q, np.ones((q.shape[0], 1), np.float32)], 1)

    return cm, sm, cloud(cm), cloud(sm), qs(cm), qs(sm)


def restate(drv, knn_drv, kind, cloud, q_sensor, twist):
    """The fp32 restatement per query: neighbours in the checker's search order at pointAssociateToMap(q)."""
    qm = mr.Pose(twist).to_map(q_sensor)
    n = q_sensor.shape[0]
    sel = np.zeros(n, np.int8)
    coeff = np.zeros((n, 4), np.float32)
    if n == 0 or cloud.shape[0] < 5:
        return sel, coeff, qm
    idx, d2 = knn_drv.knn(cloud, qm, 5)
    fit = fr.map_corner_fit if kind == "corner" else fr.map_surf_fit
    for i in range(n):
        if d2[i, 4] < 1.0:
            s, c = fit(drv, cloud[idx[i], :3], qm[i, :3])
            sel[i], coeff[i] = s, c
    return sel, coeff, qm


def assert_same(sel, coeff, ref_sel, ref_coeff, names, what):
    bad = (sel != ref_sel) | ~fr.same_bits(coeff, ref_coeff)
    assert not bad.any(), (f"{what}: {bad.sum()} differ, first {[names[i] for i in np.flatnonzero(bad)[:5]]}: "
                           f"{coeff[bad][:3]} sel {sel[bad][:3]} vs {ref_coeff[bad][:3]} sel {ref_sel[bad][:3]}")


# ---------------------------------------------------------------------------------------------- the catalogue's reach
def test_catalogue_reaches_its_branches(oracle, catalogue):
    fam = {}
    for c in catalogue:
        fam.setdefault(c.family, []).append(c)
    for c in catalogue:
        if c.kind == "corner":
            m2, v = fr.eigen_v1norm2(c.pts)
            if c.family in ("collinear_axis", "planar", "axis_ties", "ev_ratio_edge", "query_on_line", "identical") \
                    and c.name != "corner_planar_random":
                assert v <= fr.FLT_MIN, c.name   # closed-form tridiagonalisation shortcut
            if c.family == "m2_tiny":
                assert m2 != 0 and v <= fr.FLT_MIN, (c.name, m2, v)
            if c.family in ("collinear_general", "random", "far_3km", "tiny_spread"):
                assert v > fr.FLT_MIN, c.name
        else:
            br, x = fr.colpiv_branches(c.pts)
            np.testing.assert_array_equal(x.view(np.uint32), oracle.lsq53(c.pts).view(np.uint32), err_msg=c.name)
            if c.family in ("collinear", "origin_plane"):
                assert br["nonzero"] == 2, (c.name, br)
            if c.family == "identical":
                assert br["nonzero"] == 1, (c.name, br)
            if c.family == "pivot_ties":
                assert br["pivot_tie"], (c.name, br)
            if c.family == "near_parallel":
                assert br["recomputed"] >= 1, (c.name, br)
    # the three fp32 edges of the line test, and the 0.2 / 0.1 edges of the plane test, on the stated side
    ev = {c.name: oracle.eig_sym(fr.corner_covariance(c.pts)[1])[0] for c in fam["ev_ratio_edge"]}
    e = ev["corner_ev_ratio_eq"]
    assert e[2] == np.float32(3) * e[1]
    e = ev["corner_ev_ratio_above"]
    assert e[2] == np.nextafter(np.float32(3) * e[1], np.float32(np.inf))
    e = ev["corner_ev_ratio_below"]
    assert e[2] == np.nextafter(np.float32(3) * e[1], np.float32(-np.inf))
    got = {c.name: fr.map_surf_fit(oracle, c.pts, c.q) for c in fam["valid_edge"] + fam["s_edge"]}
    assert not got["surf_valid_at_0.2f"][0] and not got["surf_valid_at_0.2f"][1].any()
    assert got["surf_valid_below_0.2f"][1].any()
    assert got["surf_s_above_0.1"][0] and not got["surf_s_below_0.1"][0] and got["surf_s_below_0.1"][1].any()
    # query on the line: a012 = 0 -> NaN coefficient, ld2 = 0 -> s = 1 -> selected (as the reference does)
    for c in fam["query_on_line"]:
        s, co = fr.map_corner_fit(oracle, c.pts, c.q)
        assert s and np.isnan(co[:3]).all() and co[3] == 0, (c.name, co)
    s, co = fr.map_surf_fit(oracle, fam["origin_points"][0].pts, fam["origin_points"][0].q)
    assert not s and np.isnan(co).all()
    for c in fr.tie_cases():
        assert sum(1 for _ in fr.ordered_alternatives(c.pts, c.q)) > 1, c.name


# ---------------------------------------------------------------------------------------------- fp32 vs the checker
@pytest.mark.parametrize("pose", ["zero", "yaw"])
def test_map_fits_equal_checker_on_catalogue(oracle, catalogue, pose):
    from oracle import pydriver
    twist = ZERO if pose == "zero" else YAW
    for name, group in batches(catalogue + fr.tie_cases()).items():
        cm, sm, cmap, smap, cq, sq = batch_clouds(group, twist)
        ref = pydriver.map_iteration(oracle, cmap if cmap.shape[0] else np.zeros((0, 4), np.float32),
                                     smap, cq, sq, twist)
        sel_c, co_c, _ = restate(oracle, oracle, "corner", cmap, cq, twist)
        sel_s, co_s, _ = restate(oracle, oracle, "surf", smap, sq, twist)
        sel = np.concatenate([sel_c, sel_s])
        coeff = np.concatenate([co_c, co_s])
        names = [c.name for c in cm + sm]
        assert_same(sel, coeff, ref["selected"], ref["coeff"], names, f"batch {name}, pose {pose}")
        if pose == "zero":  # the designed neighbour order is the search order
            for i, c in enumerate(cm + sm):
                if c.family == "ties":
                    continue
                fit = fr.map_corner_fit if c.kind == "corner" else fr.map_surf_fit
                s, co = fit(oracle, c.pts, c.q)
                assert s == sel[i] and fr.same_bits(co[None], coeff[i:i + 1])[0], c.name


@pytest.fixture(scope="module")
def vlp16_map_queries(oracle, scene):
    from loam_velodyne_b200 import synth
    pts, rs = synth.make_sweep(scene, synth.Lidar.vlp16(), 5, yaw_rate=math.radians(5.0))
    s = oracle.scanreg()
    s.process(pts, rs)
    cq = oracle.voxel_grid(s.cloud("less_sharp"), 0.2)
    sq = oracle.voxel_grid(s.cloud("less_flat"), 0.4)
    pos, yaw = synth.pose_at(0.6, np.array([0.0, 0.0, 1.0]), math.radians(5.0))
    twists = [np.asarray(t, np.float32) for t in
              ((0.0, yaw, 0.0, *pos), (0.002, yaw + 0.004, -0.003, pos[0] + 0.05, pos[1] - 0.02, pos[2] + 0.08))]
    return cq, sq, twists


def test_map_fits_equal_checker_on_sweep(oracle, map_200k, vlp16_map_queries):
    from oracle import pydriver
    corner, surf = map_200k
    cq, sq, twists = vlp16_map_queries
    for twist in twists:
        ref = pydriver.map_iteration(oracle, corner, surf, cq, sq, twist)
        sel_c, co_c, _ = restate(oracle, oracle, "corner", corner, cq, twist)
        sel_s, co_s, _ = restate(oracle, oracle, "surf", surf, sq, twist)
        sel, coeff = np.concatenate([sel_c, sel_s]), np.concatenate([co_c, co_s])
        assert ref["n_selected"] > 200
        assert_same(sel, coeff, ref["selected"], ref["coeff"], list(range(sel.shape[0])), f"VLP-16 sweep at {twist}")


def odom_restate(cs, exp, ind, it, nq_sharp, nq_flat):
    """Restated coefficients of the odometry catalogue at iteration `it`, using the correspondence indices `ind`."""
    lines = [c for c in cs if c.kind == "corner"]
    planes = [c for c in cs if c.kind == "surf"]
    sel = np.zeros(nq_sharp + nq_flat, np.int8)
    coeff = np.zeros((nq_sharp + nq_flat, 4), np.float32)
    for i, c in enumerate(lines):
        s, co = fr.odom_corner_fit(c.pts[0], c.pts[1], c.q, it)
        sel[i], coeff[i] = s, co
    for i, c in enumerate(planes):
        s, co = fr.odom_surf_fit(c.pts[0], c.pts[1], c.pts[2], c.q, it)
        sel[nq_sharp + i], coeff[nq_sharp + i] = s, co
    return sel, coeff


def odom_rows(cs, nq_sharp):
    lines = [c for c in cs if c.kind == "corner"]
    planes = [c for c in cs if c.kind == "surf"]
    return [(i, c) for i, c in enumerate(lines)] + [(nq_sharp + i, c) for i, c in enumerate(planes)]


def check_odom_indices(cs, exp, ind, nq_sharp, what):
    for row, c in odom_rows(cs, nq_sharp):
        e = exp[c.name]
        if c.tie_pair:  # t1 == t2: the closest point is either copy
            assert sorted(ind[row, :2].tolist()) == sorted(e[:2]) and ind[row, 2] == e[2], (what, c.name, ind[row], e)
        else:
            assert tuple(ind[row].tolist()) == e, (what, c.name, ind[row], e)
    rows = {r for r, _ in odom_rows(cs, nq_sharp)}
    pad = np.array([r not in rows for r in range(ind.shape[0])])
    assert (ind[pad, 0] == -1).all(), what


@pytest.mark.parametrize("twist_name", ["zero", "twist"])
def test_odom_fits_equal_checker_on_catalogue(oracle, twist_name):
    from oracle import pydriver
    tw = ZERO if twist_name == "zero" else TWIST
    allc = fr.odom_cases(0)
    for batch in ("finite", "poison"):
        cs = [c for c in allc if c.batch == batch]
        lc, ls, sharp, flat, exp = fr.odom_clouds(cs)
        it_ = pydriver.OdomIterator(oracle, lc, ls, sharp, flat)
        for it in (0, 4, 5, 9):
            ref = it_.iterate(it, tw)
            check_odom_indices(cs, exp, ref["ind"], sharp.shape[0], f"{batch} iteration {it}")
            sel, coeff = odom_restate(cs, exp, ref["ind"], it, sharp.shape[0], flat.shape[0])
            names = [""] * sel.shape[0]
            for r, c in odom_rows(cs, sharp.shape[0]):
                names[r] = c.name
            assert_same(sel, coeff, ref["selected"], ref["coeff"], names, f"odometry {batch}, iteration {it}")
            finite = np.isfinite(ref["AtA"]).all() and np.isfinite(ref["AtB"]).all()
            assert finite == (batch == "finite" or it >= 5), (batch, it)
    # what the poison batch is for: below iteration 5 the NaN rows are selected
    cs = [c for c in allc if c.batch == "poison"]
    assert all(fr.odom_corner_fit(c.pts[0], c.pts[1], c.q, 0)[0] for c in cs if c.kind == "corner")
    assert all(fr.odom_surf_fit(c.pts[0], c.pts[1], c.pts[2], c.q, 0)[0] for c in cs if c.kind == "surf")
    edges = {c.name: c for c in allc if c.family == "weight_edge"}
    for kind in ("line", "plane"):
        a, b = edges[f"odom_{kind}_weight_above"], edges[f"odom_{kind}_weight_below"]
        fit = (lambda c, it: fr.odom_corner_fit(c.pts[0], c.pts[1], c.q, it)) if kind == "line" else \
            (lambda c, it: fr.odom_surf_fit(c.pts[0], c.pts[1], c.pts[2], c.q, it))
        assert fit(a, 4)[0] and fit(b, 4)[0] and fit(a, 5)[0] and not fit(b, 5)[0], kind


def odom_sweep(oracle, scene):
    from loam_velodyne_b200 import synth
    lidar = synth.Lidar.vlp16()
    p0, r0 = synth.make_sweep(scene, lidar, 0, yaw_rate=math.radians(5.0))
    p1, r1 = synth.make_sweep(scene, lidar, 1, yaw_rate=math.radians(5.0))
    s = oracle.scanreg()
    s.process(p0, r0)
    last_c, last_s = s.cloud("less_sharp").copy(), s.cloud("less_flat").copy()
    last_c[:, 3] = np.floor(last_c[:, 3])
    last_s[:, 3] = np.floor(last_s[:, 3])
    s.process(p1, r1)
    return last_c, last_s, s.cloud("sharp"), s.cloud("flat")


def odom_restate_ind(lc, ls, sharp, flat, ind, it):
    """The fp32 restatement of every query at the given correspondence indices (zero twist: toStart is exact)."""
    ns = sharp.shape[0]
    n = ns + flat.shape[0]
    sel = np.zeros(n, np.int8)
    coeff = np.zeros((n, 4), np.float32)
    for i in range(n):
        i1, i2, i3 = ind[i]
        if i < ns and i2 >= 0:
            sel[i], coeff[i] = fr.odom_corner_fit(lc[i1], lc[i2], sharp[i], it)
        elif i >= ns and i2 >= 0 and i3 >= 0:
            sel[i], coeff[i] = fr.odom_surf_fit(ls[i1], ls[i2], ls[i3], flat[i - ns], it)
    return sel, coeff


def test_odom_fits_equal_checker_on_sweep(oracle, scene):
    from oracle import pydriver
    lc, ls, sharp, flat = odom_sweep(oracle, scene)
    it_ = pydriver.OdomIterator(oracle, lc, ls, sharp, flat)
    for it in (0, 4, 5, 9):
        ref = it_.iterate(it, ZERO)
        sel, coeff = odom_restate_ind(lc, ls, sharp, flat, ref["ind"], it)
        assert ref["n_selected"] > 100
        assert_same(sel, coeff, ref["selected"], ref["coeff"], list(range(sel.shape[0])), f"VLP-16 iteration {it}")


# ---------------------------------------------------------------------------------------------- fp32 vs float64
def compare64(drv, kind, nn, q):
    """-> (compared, error / bar) for one correspondence; compared is False when a decision is within 1e-6 of its
    threshold or the problem is too ill-conditioned for any bar (cond * eps32 > 1e-2)."""
    fit32 = fr.map_corner_fit if kind == "corner" else fr.map_surf_fit
    fit64 = fr.map_corner_fit64 if kind == "corner" else fr.map_surf_fit64
    s32, c32 = fit32(drv, nn, q)
    s64, c64, margins, cond = fit64(nn, q)
    if fr.near_threshold(margins) or not np.isfinite(cond) or cond * fr.EPS32 > 1e-2:
        return False, 0.0
    assert s32 == s64, (kind, margins, cond)
    if not s32:
        return True, 0.0
    k = K_CORNER if kind == "corner" else K_SURF
    err = np.abs(c32.astype(np.float64) - c64) / np.maximum(1.0, np.abs(c64))
    return True, float(err.max() / (k * fr.EPS32 * cond))


def test_fp32_agrees_with_float64(oracle, catalogue, map_200k, vlp16_map_queries):
    worst, n_cmp, skipped = 0.0, 0, []
    for c in catalogue:
        ok, r = compare64(oracle, c.kind, c.pts, c.q)
        if ok:
            n_cmp += 1
            worst = max(worst, r)
        else:
            skipped.append(c.name)
    corner, surf = map_200k
    cq, sq, twists = vlp16_map_queries
    for kind, cloud, q in (("corner", corner, cq), ("surf", surf, sq)):
        qm = mr.Pose(twists[0]).to_map(q)
        idx, d2 = oracle.knn(cloud, qm, 5)
        for i in np.flatnonzero(d2[:, 4] < 1.0):
            ok, r = compare64(oracle, kind, cloud[idx[i], :3], qm[i, :3])
            n_cmp += ok
            worst = max(worst, r)
    print(f"float64 comparison: {n_cmp} fits, worst error / bar {worst:.3g}; not compared: {skipped}")
    assert n_cmp > 1000
    assert worst <= 1.0
