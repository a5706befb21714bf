"""Every compiled copy of the per-correspondence line and plane fits against the fp32 restatement of
tests/fit_reference.py (pinned to the checker by test_fit_reference.py), bit for bit and NaN-aware, with no slack:
map_iterate_kernel over the bounding-box grid (GridCellLookup) and over the pipeline's persistent store
(MapCellLookup), and the odometry iteration kernel through both of its entry paths.  The inputs are
the catalogue of degenerate neighbourhoods of fit_reference.cases / odom_cases and the real sweeps of the existing
per-correspondence tests, restricted there to queries whose search has no exact distance tie."""
import contextlib
import math

import numpy as np
import pytest

import fit_reference as fr
import map_reference as mr
from test_fit_reference import (TWIST, YAW, ZERO, batch_clouds, batches, check_odom_indices, odom_restate,
                                odom_restate_ind, odom_rows, odom_sweep, restate)

pytestmark = pytest.mark.gpu
LEAVES = (0.2, 0.4)


@contextlib.contextmanager
def _ctx():
    from loam_velodyne_b200 import api
    c = api.Ctx(0)
    try:
        yield c
    finally:
        c.close()


def _all125(twist, cen0=(10, 5, 10)):
    """The 125 cubes around the pose (test_map_stage.py's "all125" window)."""
    cen, _, _ = mr.window(twist, cen0)
    p = np.asarray(twist[3:], np.float64)
    centre = [int((p[a] + 25.0) / 50.0) + cen[a] - (1 if p[a] + 25.0 < 0 else 0) for a in range(3)]
    cubes = [i + mr.W * j + mr.W * mr.H * k
             for i in range(centre[0] - 2, centre[0] + 3) for j in range(centre[1] - 2, centre[1] + 3)
             for k in range(centre[2] - 2, centre[2] + 3)
             if 0 <= i < mr.W and 0 <= j < mr.H and 0 <= k < mr.D]
    return cen, cubes


def _expected(oracle, group, cmap, smap, cq, sq, twist):
    """Restated (sel, coeff) and, per query, every acceptable (sel, coeff): one per ordering of exactly tied
    neighbours."""
    sel_c, co_c, qmc = restate(oracle, oracle, "corner", cmap, cq, twist)
    sel_s, co_s, qms = restate(oracle, oracle, "surf", smap, sq, twist)
    sel, coeff = np.concatenate([sel_c, sel_s]), np.concatenate([co_c, co_s])
    alts = {}
    for i, (kind, cloud, qm) in enumerate([("corner", cmap, q) for q in qmc] + [("surf", smap, q) for q in qms]):
        _, d2 = oracle.knn(cloud, qm[None], 6)
        d = d2[0][d2[0] < 1.0]
        if np.any(d[1:] == d[:-1]):  # a tie among the neighbours within 1 m
            idx, _ = oracle.knn(cloud, qm[None], 5)
            fit = fr.map_corner_fit if kind == "corner" else fr.map_surf_fit
            alts[i] = [fit(oracle, p, qm[:3]) for p in fr.ordered_alternatives(cloud[idx[0], :3], qm[:3])]
    return sel, coeff, alts


def _check_map(got, exp, names, what):
    ne, coeff, sel = got
    e_sel, e_coeff, alts = exp
    bad = (sel != e_sel) | ~fr.same_bits(coeff, e_coeff)
    for i in np.flatnonzero(bad):
        if i in alts and any(bool(s) == bool(sel[i]) and fr.same_bits(c[None], coeff[i:i + 1])[0] for s, c in alts[i]):
            bad[i] = False
    assert not bad.any(), (f"{what}: {[names[i] for i in np.flatnonzero(bad)[:6]]} differ: {coeff[bad][:3]} "
                           f"sel {sel[bad][:3]} vs {e_coeff[bad][:3]} sel {e_sel[bad][:3]}")
    finite = bool(np.isfinite(e_coeff[e_sel == 1]).all())
    assert bool(np.isfinite(ne["AtA"]).all() and np.isfinite(ne["AtB"]).all()) == finite, what
    assert int(round(ne["n_selected"])) == int(e_sel.sum()), what


# ---------------------------------------------------------------------------------------------- mapping: grid path
def grid_checks(oracle, catalogue, poses):
    from loam_velodyne_b200 import api
    n = 0
    with _ctx() as c:
        for pose in poses:
            twist = ZERO if pose == "zero" else YAW
            for name, group in batches(catalogue + fr.tie_cases()).items():
                cm, sm, cmap, smap, cq, sq = batch_clouds(group, twist)
                c.tree_build(api.TREE_MAP_CORNER, cmap)
                c.tree_build(api.TREE_MAP_SURF, smap)
                c.map_set_queries(cq, sq)
                got = c.map_iterate(twist, debug=True)
                exp = _expected(oracle, group, cmap, smap, cq, sq, twist)
                _check_map(got, exp, [g.name for g in cm + sm], f"grid path, batch {name}, pose {pose}")
                n += len(group)
    return n


@pytest.mark.parametrize("pose", ["zero", "yaw"])
def test_grid_path_catalogue(oracle, pose):
    cat = fr.cases(0, oracle)
    assert grid_checks(oracle, cat, [pose]) == len(cat) + len(fr.tie_cases())


# ---------------------------------------------------------------------------------------------- mapping: store path
def store_checks(oracle, catalogue):
    """The catalogue through map_pool_append / the stack slots / map_begin_sweep at the zero pose (the stack round
    trip is then exact), with cell pruning off and on.  The 3 km clusters lie outside the 125 cubes and are left out."""
    from loam_velodyne_b200 import api
    n = 0
    cen, valid = _all125(ZERO)
    for name, group in batches(catalogue + fr.tie_cases()).items():
        if name == "far":
            continue
        cm, sm, cmap, smap, cq, sq = batch_clouds(group, ZERO)
        # one mark per query (the intensity survives the 0.2 / 0.4 m voxel filter of a lone point)
        cq[:, 3] = 100.0 + np.arange(cq.shape[0])
        sq[:, 3] = 100.0 + np.arange(sq.shape[0])
        with _ctx() as c:
            for kind, pts in ((0, cmap), (1, smap)):
                if pts.shape[0]:
                    c.map_pool_append(kind, pts)
            c.cloud_upload(api.C_MAP_CORNER_LAST, cq)
            c.cloud_upload(api.C_MAP_SURF_LAST, sq)
            sizes = c.map_begin_sweep(ZERO, cen, valid, *LEAVES)
            stacks = (c.cloud_download(api.C_MAP_CORNER_STACK_DS), c.cloud_download(api.C_MAP_SURF_STACK_DS))
            assert sizes[2] == cq.shape[0] and sizes[3] == sq.shape[0], (name, sizes)
            for st, q in zip(stacks, (cq, sq)):
                o = np.argsort(st[:, 3])
                np.testing.assert_array_equal(st[o], q, err_msg=f"{name}: stack round trip")
            exp = _expected(oracle, group, cmap, smap, stacks[0], stacks[1], ZERO)
            names_c = [g.name for g in cm]
            names_s = [g.name for g in sm]
            names = [names_c[int(m) - 100] for m in stacks[0][:, 3]] + [names_s[int(m) - 100] for m in stacks[1][:, 3]]
            for prune in (0, 1):
                c.debug_map_prune(prune)
                got = c.map_iterate(ZERO, debug=True)
                _check_map(got, exp, names, f"store path, batch {name}, prune {prune}")
        n += len(group)
    return n


def test_store_path_catalogue(oracle):
    cat = fr.cases(0, oracle)
    assert store_checks(oracle, cat) == len([c for c in cat if c.batch != "far"]) + len(fr.tie_cases())


# ---------------------------------------------------------------------------------------------- odometry
@pytest.mark.parametrize("path", ["set_last", "cloud_slots"])
def test_odom_catalogue(path):
    from loam_velodyne_b200 import api
    allc = fr.odom_cases(0)
    for batch in ("finite", "poison"):
        cs = [c for c in allc if c.batch == batch]
        lc, ls, sharp, flat, exp = fr.odom_clouds(cs)
        ns = sharp.shape[0]
        names = [""] * (ns + flat.shape[0])
        for r, c in odom_rows(cs, ns):
            names[r] = c.name
        with _ctx() as c:
            if path == "set_last":
                c.odom_set_last(lc, ls)
                c.odom_set_current(sharp, flat)
            else:
                c.cloud_upload(api.C_ODOM_LAST_CORNER, lc)
                c.cloud_upload(api.C_ODOM_LAST_SURF, ls)
                c.odom_rebuild_last()
                c.cloud_upload(api.C_ODOM_SHARP, sharp)
                c.cloud_upload(api.C_ODOM_FLAT, flat)
                c.odom_prepare()
            for tw in (ZERO, TWIST):
                for it in (0, 4, 5, 9):
                    ne, coeff, sel, ind = c.odom_iterate(tw, it, debug=True)
                    what = f"odometry {path}, {batch}, twist {tw[0]}, iteration {it}"
                    check_odom_indices(cs, exp, ind, ns, what)
                    e_sel, e_coeff = odom_restate(cs, exp, ind, it, ns, flat.shape[0])
                    bad = (sel != e_sel) | ~fr.same_bits(coeff, e_coeff)
                    assert not bad.any(), (what, [names[i] for i in np.flatnonzero(bad)], coeff[bad], e_coeff[bad])
                    finite = bool(np.isfinite(e_coeff[e_sel == 1]).all())
                    assert bool(np.isfinite(ne["AtA"]).all() and np.isfinite(ne["AtB"]).all()) == finite, what
                    assert finite == (batch == "finite" or it >= 5), what


# ---------------------------------------------------------------------------------------------- real sweeps, no slack
def _no_tie(oracle, cloud, qm):
    """Queries whose 6 nearest points within 1 m have no exact distance tie."""
    _, d2 = oracle.knn(cloud, qm, 6)
    eq = (d2[:, 1:] == d2[:, :-1]) & (d2[:, :-1] < 1.0)
    return ~eq.any(axis=1)


@pytest.mark.parametrize("lidar", ["vlp16", "hdl64"])
def test_map_real_sweep_exact(oracle, scene, map_200k, lidar):
    """The sweeps of test_map_iteration_per_correspondence (and an HDL-64 one): exact on every query whose search is
    unambiguous, over the grid and over the store."""
    from loam_velodyne_b200 import api, synth
    corner, surf = map_200k
    pts, rs = synth.make_sweep(scene, getattr(synth.Lidar, lidar)(), 5, yaw_rate=math.radians(5.0))
    s = oracle.scanreg()
    s.process(pts, rs)
    cq = oracle.voxel_grid(s.cloud("less_sharp"), 0.2)
    sq = oracle.voxel_grid(s.cloud("less_flat"), 0.4)
    pos, yaw = synth.pose_at(0.6, np.array([0.0, 0.0, 1.0]), math.radians(5.0))
    with _ctx() as c:
        c.tree_build(api.TREE_MAP_CORNER, corner)
        c.tree_build(api.TREE_MAP_SURF, surf)
        for twist in ((0.0, yaw, 0.0, *pos), (0.002, yaw + 0.004, -0.003, pos[0] + 0.05, pos[1] - 0.02, pos[2] + 0.08)):
            twist = np.asarray(twist, np.float32)
            c.map_set_queries(cq, sq)
            ne, coeff, sel = c.map_iterate(twist, debug=True)
            e_sel_c, e_co_c, qmc = restate(oracle, oracle, "corner", corner, cq, twist)
            e_sel_s, e_co_s, qms = restate(oracle, oracle, "surf", surf, sq, twist)
            e_sel, e_coeff = np.concatenate([e_sel_c, e_sel_s]), np.concatenate([e_co_c, e_co_s])
            clean = np.concatenate([_no_tie(oracle, corner, qmc), _no_tie(oracle, surf, qms)])
            assert clean.mean() > 0.95 and e_sel[clean].sum() > 200
            bad = clean & ((sel != e_sel) | ~fr.same_bits(coeff, e_coeff))
            assert not bad.any(), (lidar, twist, np.flatnonzero(bad)[:10], coeff[bad][:3], e_coeff[bad][:3])
            # the rest keeps the bar of test_map_iteration_per_correspondence
            assert int((sel != e_sel).sum()) <= 2


def test_odom_real_sweep_exact(oracle, scene):
    """The sweep pair of test_odom_iteration_per_correspondence at zero twist: on every query without a 1-NN tie the
    indices equal the checker's and the coefficients the restatement's."""
    from oracle import pydriver
    lc, ls, sharp, flat = odom_sweep(oracle, scene)
    it_ = pydriver.OdomIterator(oracle, lc, ls, sharp, flat)
    ns = sharp.shape[0]
    _, dc = oracle.knn(lc, sharp, 2)
    _, dsf = oracle.knn(ls, flat, 2)
    clean = np.concatenate([dc[:, 0] != dc[:, 1], dsf[:, 0] != dsf[:, 1]])
    assert clean.mean() > 0.95
    with _ctx() as c:
        c.odom_set_last(lc, ls)
        c.odom_set_current(sharp, flat)
        for it in (0, 4, 5, 9):
            ref = it_.iterate(it, ZERO)
            ne, coeff, sel, ind = c.odom_iterate(ZERO, it, debug=True)
            bad = clean & (ind != ref["ind"]).any(axis=1)
            assert not bad.any(), (it, np.flatnonzero(bad)[:10])
            e_sel, e_coeff = odom_restate_ind(lc, ls, sharp, flat, ind, it)
            bad = clean & ((sel != e_sel) | ~fr.same_bits(coeff, e_coeff))
            assert not bad.any(), (it, np.flatnonzero(bad)[:10], coeff[bad][:3], e_coeff[bad][:3])
            assert ref["n_selected"] > 100 and ns > 0
