"""The restatement of snapshots and merging (tests/merge_reference.py) on its own: resume is exact, a zero pose equals
none, counts are conserved, a merge under a pose agrees with inserting the transformed points, and every hand-made
case is told apart from a deliberately wrong restatement.  CPU only."""
import math

import numpy as np
import pytest

import align_reference as ar
import dense_reference as dr
import merge_reference as mr
import visibility_reference as vr


def same_state(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a.state(), b.state()))


@pytest.fixture(scope="module")
def runs(scene):
    from loam_velodyne_b200 import synth
    return {"vlp16": vr.moving_box_run(scene, synth.Lidar.vlp16(n_az=900), 6),
            "hdl64": vr.moving_box_run(scene, synth.Lidar.hdl64(n_az=512), 4)}


def restated(run, leaf, evidence=True):
    ref = mr.MergeMapRef(leaf, h_res=0.4 if evidence else 0.0, v_res=0.4, margin=0.5)
    for pts, twist, _ in run:
        ref.sweep(pts, twist)
    return ref


@pytest.mark.parametrize("leaf", [0.1, 0.2, 0.4])
@pytest.mark.parametrize("lidar", ["vlp16", "hdl64"])
def test_resume_is_exact(runs, lidar, leaf):
    """Snapshot -> merge into an empty map of the same leaf with no pose gives the same state, evidence included; the
    rest of the run inserted afterwards gives the uninterrupted run's map."""
    run = runs[lidar]
    whole = restated(run, leaf)
    assert whole.misses.sum() > 0 and whole.hits.max() > 1  # evidence of both kinds is carried
    half = restated(run[:len(run) // 2], leaf)
    resumed = mr.MergeMapRef(leaf, h_res=0.4, v_res=0.4, margin=0.5)
    got = resumed.merge(half.snapshot())
    assert got["new"] == int(half.count.sum()) and got["stored"] == got["skipped"] == got["dropped"] == 0
    assert same_state(resumed, half)
    for pts, twist, _ in run[len(run) // 2:]:
        resumed.sweep(pts, twist)
    assert same_state(resumed, whole)


def test_zero_pose_equals_none(runs):
    snap = restated(runs["vlp16"], 0.2).snapshot()
    assert not np.any(np.signbit(snap["sums"]) & (snap["sums"] == 0.0))  # no stored sum is -0.0
    a, b = mr.MergeMapRef(0.2), mr.MergeMapRef(0.2)
    a.merge(snap)
    b.merge(snap, np.zeros(6, np.float32))
    assert same_state(a, b)


@pytest.mark.parametrize("twist", [None, (0.02, 1.1, -0.03, 3.5, -0.4, 12.25), (0.0, 0.0, 0.0, 524200.0, 0.0, 0.0)])
def test_counts_are_conserved(runs, twist):
    """Counts merged in = counts added to stored voxels + the new voxels' counts + skipped + dropped; the map's count
    total grows by the first two."""
    snap = restated(runs["hdl64"], 0.1).snapshot()
    ref = restated(runs["vlp16"], 0.2)
    ref.max_voxels = ref.keys.size + 1000
    before = int(ref.count.sum())
    got = ref.merge(snap, twist)
    assert got["stored"] + got["new"] + got["skipped"] + got["dropped"] == int(snap["counts"].astype(np.int64).sum())
    assert int(ref.count.sum()) == before + got["stored"] + got["new"]
    if twist is None:
        assert got["dropped"] > 0 and ref.keys.size == ref.max_voxels


@pytest.mark.parametrize("twist", [(0.0, 0.7, 0.0, 1.3, 0.0, -2.2), (0.05, -2.4, 0.02, -7.9, 0.3, 4.05)])
def test_pose_agrees_with_transformed_points(scene, twist):
    """Each merged entry's destination voxel lies in the bounding box of the voxels its transformed points occupy (the
    centroid is in their hull and floorf is monotone); an entry whose centroid lies within rounding of a voxel face may
    land one voxel beyond."""
    from loam_velodyne_b200 import synth
    leaf = 0.2
    pts, _ = synth.make_sweep(scene, synth.Lidar.vlp16(n_az=900), 0, yaw_rate=math.radians(5.0))
    ref = mr.MergeMapRef(leaf)
    ref.insert(pts)
    snap = ref.snapshot()
    k = dr.voxel_keys(pts, leaf)
    t = np.asarray(twist, np.float32)
    moved = ar.to_map64(t.astype(np.float64), pts[:, :3].astype(np.float64)) + t[3:].astype(np.float64)
    vox = dr.key_voxel(dr.voxel_keys(np.concatenate([moved.astype(np.float32), pts[:, 3:]], axis=1), leaf))
    ok = k != dr.EMPTY
    order = np.argsort(k[ok], kind="stable")
    sk, sv = k[ok][order], vox[ok][order]
    start = np.searchsorted(sk, snap["keys"])
    end = np.searchsorted(sk, snap["keys"], side="right")
    lo = np.minimum.reduceat(sv, start, axis=0)
    hi = np.maximum.reduceat(sv, start, axis=0)
    assert np.array_equal(end - start, snap["counts"])
    S2 = mr.transform_sums(snap["counts"], snap["sums"], t)
    dest = dr.key_voxel(mr.destination_keys(snap["counts"], S2, leaf))
    g = (S2[:, :3] / snap["counts"][:, None].astype(np.float64)) * float(np.float32(1.0) / np.float32(leaf))
    near = np.abs(g - np.round(g)) < 1e-5
    inside = (dest >= lo) & (dest <= hi)
    assert np.all(inside | (near & (dest >= lo - 1) & (dest <= hi + 1)))
    assert inside.all(axis=1).mean() > 0.999


def test_hand_cases_and_wrong_variants():
    """Every hand-made case changes under at least one wrong restatement, and every wrong restatement is caught by at
    least one case."""
    caught = {v: [] for v in mr.VARIANTS}
    for name, case in mr.hand_cases().items():
        good = mr.run_case(case)
        changed = []
        for v in mr.VARIANTS:
            if not same_state(good, mr.run_case(case, v)):
                caught[v].append(name)
                changed.append(v)
        assert changed, name
    assert all(caught.values()), caught


def test_hand_case_details():
    cases = mr.hand_cases()
    abc, cba = mr.run_case(cases["one_voxel_order_abc"]), mr.run_case(cases["one_voxel_order_cba"])
    assert abc.keys.size == cba.keys.size == 1 and abc.S[0, 0] == 1.0 and cba.S[0, 0] > 1.0
    assert same_state(mr.run_case(cases["two_entries_ab"]), mr.run_case(cases["two_entries_ba"]))
    face = mr.run_case(cases["face"])
    assert [int(v) for v in dr.key_voxel(face.keys)[:, 0]] == [2, 3] and face.count.tolist() == [1, 7]
    sat = mr.run_case(cases["saturation"])
    assert sat.hits.tolist() == [65535, 65535, 65534] and sat.misses.tolist() == [65535, 65535, 2]
    kr = mr.run_case(cases["key_range"])
    assert kr.skipped == 1 and kr.keys.size == 2
    cap = mr.run_case(cases["cap"])
    assert cap.keys.size == 5 and cap.dropped == 3
    assert [int(v) for v in dr.key_voxel(cap.keys)[:, 0]] == [0, 2, 4, 6, 10]


def test_argument_validation():
    """The restatement refuses what the library refuses with LOAM_B200_ERR_ARG, and a refused merge changes nothing."""
    good = mr.entries([(1, 1, 0, 0.1, 0.1, 0.1, 1.0), (2, 3, 1, 0.3, 0.3, 0.3, 2.0)])
    ref = mr.MergeMapRef(0.5)
    ref.merge(good)
    before = ref.state()
    bad = []
    for field, i, value in (("counts", 1, 0), ("hits", 0, 0), ("sums", (1, 2), np.nan), ("sums", (0, 3), np.inf),
                            ("sums", (0, 0), -np.inf)):
        s = {k: np.array(v, copy=True) if v is not None else None for k, v in good.items()}
        s[field][i] = value
        bad.append((s, None))
    bad += [(good, (0.0, np.nan, 0.0, 0.0, 0.0, 0.0)), (good, (0.0, 0.0, 0.0, np.inf, 0.0, 0.0))]
    for s, twist in bad:
        with pytest.raises(ValueError):
            ref.merge(s, twist)
    assert all(np.array_equal(x, y) for x, y in zip(before, ref.state()))
    assert ref.merge(mr.entries(np.zeros((0, 7)))) == {"stored": 0, "new": 0, "skipped": 0, "dropped": 0}
