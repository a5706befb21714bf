"""CPU: the numpy restatement of the ground calls (tests/ground_reference.py) against brute force, on hand-made targets
and clouds with known answers, against deliberately wrong restatements, and on the city scene against its ground
truth."""
import math

import numpy as np
import pytest

import align_reference as ar
import dense_reference as dr
import ground_reference as gr
import segment_reference as sr

F = np.float32
LEAF = 0.1
UP = (0.0, 1.0, 0.0, 0.0)
IDENTITY = np.zeros(6, np.float32)


def strip(x0, n, y, z=0.05, dx=LEAF, nrm=UP):
    """n voxels along x from x0 at height y, one per voxel, with one normal."""
    c = np.stack([x0 + dx * np.arange(n), np.full(n, y), np.full(n, z), np.ones(n)], 1).astype(np.float32)
    return c, np.tile(np.float32(nrm), (n, 1))


def target(*parts):
    """A loaded target (align_reference.Target) of (centroids, normals) parts."""
    c = np.concatenate([p[0] for p in parts])
    n = np.concatenate([p[1] for p in parts])
    return ar.loaded_target(LEAF, c, n)


def ground_of(t, prm, variant=None):
    return gr.dense_ground(t.keys, t.cent, t.nrm, LEAF, prm, variant)


def tilted(deg):
    a = math.radians(deg)
    return (-math.sin(a), math.cos(a), 0.0, 0.0)


def target_cases():
    """name -> (target, params, check(labels, ground) -> bool).  Each holds a known answer."""
    p1 = gr.Params(15.0, 0.05, 0.2, 0.2, 1)
    c = {}
    for name, deg, want in (("ramp_under", 14.9, True), ("ramp_over", 15.1, False)):
        a = math.radians(deg)
        cent, nrm = strip(0.05, 30, 0.0, nrm=tilted(deg))
        cent[:, 1] = (cent[:, 0] * math.tan(a)).astype(np.float32)
        c[name] = (target((cent, nrm)), p1, lambda lab, g, w=want: bool(g.all()) == w and bool(g.any()) == w and
                   (not w or (lab == 0).all()))
    step = F(0.2)
    for name, dy, joined in (("step_at", step, True), ("step_under", F(0.15), True),
                             ("step_ulp_over", np.nextafter(step, F(1.0)), False)):
        lower, nl = strip(0.05, 10, 0.0)
        upper, nu = strip(1.05, 10, dy)
        c[name] = (target((lower, nl), (upper, nu)), p1,
                   lambda lab, g, j=joined: g.all() and ((np.unique(lab).size == 1) == j))
    a, na = strip(0.0, 1, 0.05)
    b, nb = strip(F(0.2), 1, 0.05)  # exactly tol apart horizontally
    c["exact_tol"] = (target((a, na), (b, nb)), p1, lambda lab, g: g.all() and lab[0] == lab[1])
    floor, nf = strip(0.05, 30, 0.0)
    table, nt = strip(3.05, 8, 0.75)
    c["table"] = (target((floor, nf), (table, nt)), gr.Params(15.0, 0.05, 0.2, 0.2, 10),
                  lambda lab, g: g.sum() == 30 and (lab[g] == 0).all())
    # a box car: roof at 1.5 m with upward normals, sides with horizontal normals, floor around it
    roof, nr_ = strip(1.05, 20, 1.5)
    side0, ns0 = strip(0.95, 1, 0.8, nrm=(1.0, 0.0, 0.0, 0.0))
    side1, ns1 = strip(3.05, 1, 0.8, nrm=(1.0, 0.0, 0.0, 0.0))
    c["car"] = (target((floor, nf), (roof, nr_), (side0, ns0), (side1, ns1)), gr.Params(15.0, 0.05, 0.2, 0.2, 25),
                lambda lab, g: g.sum() == 30)
    nanf, nn = strip(0.05, 10, 0.0)
    nn[4] = np.nan
    c["nan_normal"] = (target((nanf, nn)), p1, lambda lab, g: g.sum() == 9 and lab[4] == -1 and np.unique(lab).size == 3)
    down, nd = strip(0.05, 10, 0.0, nrm=(0.0, -1.0, 0.0, 0.0))
    curved, ncv = strip(2.05, 10, 0.0, nrm=(0.0, 1.0, 0.0, 0.5))
    c["orientation_and_curvature"] = (target((down, nd), (curved, ncv)), p1,
                                      lambda lab, g: g[:10].all() and not g[10:].any())
    nanw, nw = strip(0.05, 10, 0.0, nrm=(0.0, 1.0, 0.0, np.nan))
    c["nan_w_inf"] = (target((nanw, nw)), gr.Params(15.0, np.inf, 0.2, 0.2, 1), lambda lab, g: g.all())
    c["nan_w"] = (target((nanw, nw)), p1, lambda lab, g: not g.any())
    last = F((dr.HALF - 1) * F(LEAF)) + F(0.05)
    ends = np.array([[last, 0.05, 0.05, 1.0], [-last, 0.15, 0.05, 1.0], [last - F(0.1), 0.05, 0.05, 1.0]], np.float32)
    c["key_range_ends"] = (ar.loaded_target(LEAF, ends, np.tile(np.float32(UP), (3, 1))), p1,
                           lambda lab, g: g.all() and np.unique(lab).size == 2)
    return c


@pytest.mark.parametrize("name", list(target_cases()))
def test_hand_made_targets(name):
    t, prm, check = target_cases()[name]
    lab, seg, g = ground_of(t, prm)
    assert check(lab, g), (lab.tolist(), g.tolist())
    assert seg["size"].sum() == g.sum()
    for k in range(seg["size"].size):
        assert seg["first"][k] == np.nonzero(lab == k)[0].min()


def poles_on_floor():
    """Two poles 1 m apart on a floor: one Euclidean segment through the floor, two above the ground."""
    g = np.stack(np.meshgrid(np.arange(40), np.arange(10), indexing="ij"), -1).reshape(-1, 2)
    floor = np.stack([g[:, 0] * LEAF + 0.05, np.zeros(g.shape[0]), g[:, 1] * LEAF + 0.05, np.ones(g.shape[0])], 1)
    poles = [np.array([[x, 0.05 + LEAF * (k + 1), 0.55, 1.0] for k in range(15)]) for x in (1.05, 2.05)]
    nrm = np.concatenate([np.tile(UP, (floor.shape[0], 1))] + [np.tile((1.0, 0.0, 0.0, 0.0), (15, 1))] * 2)
    return ar.loaded_target(LEAF, np.concatenate([floor] + poles).astype(np.float32), nrm.astype(np.float32))


def test_above_ground_separates_what_the_ground_joined():
    t = poles_on_floor()
    whole = sr.target_segment(t.keys, t.cent, LEAF, 0.15)
    assert whole[1]["size"].tolist() == [t.keys.size]
    _, _, g = ground_of(t, gr.Params(15.0, 0.05, 0.2, 0.2, 10))
    assert g.sum() == 400
    lab, seg = gr.segment_above_ground(t.keys, t.cent, LEAF, g, 0.15)
    assert seg["size"].tolist() == [15, 15] and (lab[g] == -1).all()


def test_above_ground_without_ground_is_dense_segment():
    t = poles_on_floor()
    _, _, g = ground_of(t, gr.Params(min_size=10**6))
    assert not g.any()
    for tol in (0.1, 0.15, 0.3):
        a = gr.segment_above_ground(t.keys, t.cent, LEAF, g, tol, 2)
        b = sr.target_segment(t.keys, t.cent, LEAF, tol, 2)
        assert np.array_equal(a[0], b[0])
        assert all(np.array_equal(a[1][f].view(np.uint8), b[1][f].view(np.uint8)) for f in b[1])


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_edges_equal_brute_force(seed):
    rng = np.random.RandomState(seed)
    v = np.unique(rng.randint(-12, 12, (1500, 3)), axis=0)
    cent = ((v + rng.uniform(0.05, 0.95, v.shape)) * LEAF).astype(np.float32)
    cent = np.concatenate([cent, np.ones((cent.shape[0], 1), np.float32)], 1)
    nrm = np.tile(np.float32(UP), (cent.shape[0], 1))
    t = ar.loaded_target(LEAF, cent, nrm)
    for prm in (gr.Params(tol=0.2, max_step=0.1), gr.Params(tol=0.1, max_step=0.3), gr.Params(tol=0.37, max_step=0.05)):
        cand = gr.candidates(t.nrm, prm)
        ii, jj = gr.ground_edges(t.keys[cand], t.cent[cand], prm, LEAF)
        idx = np.nonzero(cand)[0]
        assert set(zip(idx[ii].tolist(), idx[jj].tolist())) == gr.brute_ground_edges(t.cent, cand, prm)


def cloud_case():
    """A floor at y = 0 with a wall voxel (horizontal normal) beside it, and probe points in the map frame."""
    floor, nf = strip(0.05, 20, 0.0)
    wall, nw = strip(1.05, 1, 0.15, z=0.15, nrm=(0.0, 0.0, 1.0, 0.0))
    t = target((floor, nf), (wall, nw))
    _, _, g = ground_of(t, gr.Params(15.0, 0.05, 0.2, 0.2, 5))
    h = F(0.1)
    pts = np.array([[0.55, h, 0.05, 1.0],                          # exactly max_height above the floor: ground
                    [0.65, np.nextafter(h, F(1.0)), 0.05, 1.0],    # one ulp higher: not ground
                    [1.05, 0.12, 0.12, 1.0],                       # nearest voxel is the wall; the floor matches
                    [5.05, 0.0, 0.05, 1.0],                        # beyond the gate: not ground
                    [np.nan, 0.0, 0.0, 1.0]], np.float32)
    return t, g, pts, h


def test_cloud_hand_made():
    t, g, pts, h = cloud_case()
    assert g.sum() == 20
    lab, ng = gr.ground_cloud(t, g, pts, IDENTITY, 2, h)
    assert lab.tolist() == [1, 0, 0, 0, -1]
    assert np.array_equal(ng, pts[[1, 2, 3]])
    # the point beside the wall with a wider height band: the floor voxel is its match, 0.12 m below
    assert gr.ground_cloud(t, g, pts, IDENTITY, 2, 0.15)[0][2] == 1


def test_cloud_identity():
    """The target's own ground centroids at the zero pose are all ground at max_height = 0."""
    t = poles_on_floor()
    _, _, g = ground_of(t, gr.Params(15.0, 0.05, 0.2, 0.2, 10))
    lab, ng = gr.ground_cloud(t, g, t.cent[g], IDENTITY, 1, 0.0)
    assert (lab == 1).all() and ng.shape[0] == 0


@pytest.mark.parametrize("variant", gr.VARIANTS)
def test_wrong_restatements_are_caught(variant):
    caught = []
    for name, (t, prm, _) in target_cases().items():
        a, b = ground_of(t, prm), ground_of(t, prm, variant)
        if not (np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2])):
            caught.append(name)
    t, g, pts, h = cloud_case()
    for r, hh in ((2, h), (2, 0.15)):
        if not np.array_equal(gr.ground_cloud(t, g, pts, IDENTITY, r, hh)[0],
                              gr.ground_cloud(t, g, pts, IDENTITY, r, hh, variant)[0]):
            caught.append(f"cloud {hh}")
    assert caught, variant


# ---- the city scene: 4 HDL-64E sweeps at ground-truth poses, leaf 0.1 m, normals at radius 2, the default params.
# Measured with them: 95.2 % of the flat open ground is ground, none of the voxels above 0.3 m, and no tall
# above-ground segment spans two objects.  At tol 0.2 m and min_size 1000 (the first guess) the flat figure was 89.1 %
# (far-ground patches between rings fall under min_size) and two segments joined two buildings through that ground.
def scene_target(scene):
    from loam_velodyne_b200 import synth
    import normals_reference as nr
    from test_align_reference import MAP_TWISTS
    ref = dr.DenseMapRef(LEAF)
    for k, tw in enumerate(MAP_TWISTS):
        ref.insert(ar.static_sweep(scene, synth.Lidar.hdl64(), tw, seed=k)[1])
    cent = ref.export()[0]
    return ref.keys, cent, nr.normals(ref.keys, cent, 2, (0.0, 0.0, 0.0))


def test_scene_truth(build_libs, scene):
    keys, cent, nrm = scene_target(scene)
    x, y, z = (cent[:, a].astype(np.float64) for a in range(3))
    dists = [np.hypot(np.maximum(np.maximum(b[0] - x, x - b[1]), 0), np.maximum(np.maximum(b[4] - z, z - b[5]), 0))
             for b in scene.boxes] + [np.hypot(x - p[0], z - p[1]) - p[2] for p in scene.poles]
    D = np.stack(dists, 1)
    wall = (np.abs(x) > scene.bound - 0.5) | (np.abs(z) > scene.bound - 0.5)
    obj = np.where(D.min(axis=1) <= 0.3, D.argmin(axis=1), -1)
    obj[wall] = D.shape[1]  # the enclosing wall is one object
    flat = (np.abs(y + 1.8) <= 0.05) & (D.min(axis=1) > 1.0) & ~wall
    high = y > -1.5
    _, _, g = gr.dense_ground(keys, cent, nrm, LEAF, gr.Params())
    print(f"flat ground {g[flat].mean():.4f} of {flat.sum()}, high ground {g[high].mean():.5f} of {high.sum()}")
    assert g[flat].mean() >= 0.90
    assert g[high].mean() <= 0.01
    lab, seg = gr.segment_above_ground(keys, cent, LEAF, g, 0.2)
    tall = np.nonzero(seg["hi"][:, 1] - seg["lo"][:, 1] > 0.5)[0]
    assert tall.size > 50
    for k in tall:
        assert len(set(obj[lab == k].tolist()) - {-1}) <= 1, k
