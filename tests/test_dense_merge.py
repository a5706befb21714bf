"""Snapshots and merging of the whole-run voxel map on the GPU (csrc/densemap.cuh: dense_snapshot_kernel,
dense_merge_*_kernel; loam_b200_dense_snapshot / loam_b200_dense_merge) against the restatement
(tests/merge_reference.py) bit for bit: snapshots in the three modes, resume at any sweep, merges under poses and into
other leaves, two sessions joined through relocalisation, the drop-in and file paths, lifecycle, errors and launches."""
import math

import numpy as np
import pytest

import align_reference as ar
import dense_reference as dr
import merge_reference as mr
import visibility_reference as vr
from test_align_reference import BAR_DEG, BAR_M
from test_dense_align import map_ctx
from test_dense_carve import fresh_index

pytestmark = pytest.mark.gpu

MODES = ("map", "range", "carve")
# keys in common between B's map merged under the relocalised pose and under the true one; measured 0.667 on an H100
# 80GB HBM3 (pose error 0.25 mm, 0.026 deg: at 50 m that moves a centroid by 2 cm, a tenth of the 0.2 m leaf per axis)
SHARE_BAR = 0.6


def snap_bits(s):
    return (s["keys"], s["counts"], s["hits"], s["misses"], np.ascontiguousarray(s["sums"], np.float64).view(np.uint64))


def assert_snap(got, want, what):
    for name, a, b in zip(("keys", "counts", "hits", "misses", "sums"), snap_bits(got), snap_bits(want)):
        assert a.shape == b.shape, f"{what}: {name} shape {a.shape} vs {b.shape}"
        assert np.array_equal(a, b), f"{what}: {int((a != b).any(axis=-1).sum() if a.ndim > 1 else (a != b).sum())} " \
                                     f"{name} differ"


@pytest.fixture(scope="module")
def runs(scene):
    from loam_velodyne_b200 import synth
    return {"vlp16": vr.moving_box_run(scene, synth.Lidar.vlp16(), 8),
            "hdl64": vr.moving_box_run(scene, synth.Lidar.hdl64(n_az=1024), 5)}


def new_ctx(leaf, mode, max_voxels=2**31 - 1):
    from loam_velodyne_b200 import api
    c = api.Ctx(0)
    c.dense_enable(leaf, max_voxels)
    if mode == "range":
        c.dense_visibility(0.4, 0.4, 0.5)
    elif mode == "carve":
        c.dense_carving(0.5, 60.0)
    return c


def feed(c, run, mode):
    from loam_velodyne_b200 import api
    for pts, twist, _ in run:
        c.cloud_upload(api.C_MAP_FULL, pts)
        if mode != "map":
            c.dense_observe(api.C_MAP_FULL, twist)
        c.dense_insert(api.C_MAP_FULL)


def restated(run, leaf, max_voxels=2**31 - 1):
    """Keys, counts, sums and hits of a run (the visibility pass changes misses only)."""
    ref = mr.MergeMapRef(leaf, max_voxels)
    for pts, _, _ in run:
        ref.insert(pts)
    return ref


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("leaf", [0.1, 0.2, 0.4])
@pytest.mark.parametrize("lidar", ["vlp16", "hdl64"])
def test_snapshot(build_libs, runs, lidar, leaf, mode):
    """Keys, counts, hits and sums equal the restatement bit for bit, misses the exports'; (float)(sums / count) is the
    export's centroid."""
    c = new_ctx(leaf, mode)
    try:
        feed(c, runs[lidar], mode)
        s = c.dense_snapshot()
        want = mr.snapshot(restated(runs[lidar], leaf))
        cent, cnt, hits, misses = c.dense_export(math.inf, evidence=True)
        want["misses"] = misses
        assert_snap(s, want, f"{lidar} {leaf} {mode}")
        assert (mode == "map") == (int(misses.sum()) == 0)
        assert s["leaf"] == np.float32(leaf)
        with np.errstate(invalid="ignore"):
            c32 = (s["sums"] / s["counts"][:, None].astype(np.float64)).astype(np.float32)
        assert np.array_equal(c32.view(np.uint32), cent.view(np.uint32))
        assert np.array_equal(c.dense_export()[1], s["counts"])
    finally:
        c.close()


@pytest.mark.parametrize("mode", MODES)
def test_resume(build_libs, runs, mode):
    """Split the run at sweep k (0, the middle, the end): snapshot, merge into a fresh context with no pose, feed the
    rest -> the uninterrupted run's snapshot bit for bit; in carve mode the merged index is a fresh build's."""
    run, leaf = runs["vlp16"], 0.1
    whole = new_ctx(leaf, mode)
    try:
        feed(whole, run, mode)
        want = whole.dense_snapshot()
    finally:
        whole.close()
    for k in (0, len(run) // 2, len(run)):
        first, second = new_ctx(leaf, mode), new_ctx(leaf, mode)
        try:
            feed(first, run[:k], mode)
            part = first.dense_snapshot()
            second.dense_merge(part)
            assert_snap(second.dense_snapshot(), part, f"{mode} k {k} after the merge")
            if mode == "carve":
                bk, bm = second.dense_carve_index()
                fk, fm = fresh_index(part["keys"])
                assert np.array_equal(bk, fk) and np.array_equal(bm, fm), f"k {k}: the index is not a fresh build's"
            feed(second, run[k:], mode)
            assert_snap(second.dense_snapshot(), want, f"{mode} k {k}")
        finally:
            first.close()
            second.close()


@pytest.mark.parametrize("cap_at", ["before", "after"])
def test_resume_capped(build_libs, runs, cap_at):
    """A capped map whose cap is reached before the split, or only after it, resumes to the same map."""
    run, leaf, k = runs["vlp16"], 0.1, 4
    full = restated(run[:k], leaf).keys.size
    cap = full - 500 if cap_at == "before" else full + 2000
    assert cap < restated(run, leaf).keys.size
    whole, first, second = new_ctx(leaf, "map", cap), new_ctx(leaf, "map", cap), new_ctx(leaf, "map", cap)
    try:
        feed(whole, run, "map")
        feed(first, run[:k], "map")
        second.dense_merge(first.dense_snapshot())
        feed(second, run[k:], "map")
        got, want = second.dense_snapshot(), whole.dense_snapshot()
        assert got["keys"].size == cap
        assert_snap(got, want, f"cap reached {cap_at} the split")
        assert_snap(want, mr.snapshot(restated(run, leaf, cap)), "capped run")
    finally:
        for c in (whole, first, second):
            c.close()


def gpu_case(case):
    """A hand-made case on the GPU -> (snapshot, stats)."""
    max_voxels, initial, merged, twist = case
    c = new_ctx(mr.HAND_LEAF, "map", max_voxels)
    try:
        if initial is not None:
            c.dense_merge(initial)
        c.dense_merge(merged, twist)
        return c.dense_snapshot(), c.dense_stats()
    finally:
        c.close()


@pytest.mark.parametrize("name", list(mr.hand_cases()))
def test_hand_cases(build_libs, name):
    case = mr.hand_cases()[name]
    got, stats = gpu_case(case)
    ref = mr.run_case(case)
    assert_snap(got, ref.snapshot(), name)
    assert stats == ref.stats(), name


def merge_both(dest_ctx, ref_leaf, max_voxels, src, twist):
    """Merge src into dest_ctx and into the restatement of dest_ctx's current map (rebuilt from its snapshot: resume is
    exact) -> (GPU snapshot, restated map, where the restatement's counts went, GPU stats before and after)."""
    ref = mr.MergeMapRef(ref_leaf, max_voxels)
    ref.merge(dest_ctx.dense_snapshot())
    s0 = dest_ctx.dense_stats()
    dest_ctx.dense_merge(src, twist)
    went = ref.merge(src, twist)
    return dest_ctx.dense_snapshot(), ref, went, s0, dest_ctx.dense_stats()


def test_merge_sweep_maps(build_libs, runs):
    """Sweep maps merged under several poses, into themselves and into a larger leaf, bit for bit as restated."""
    src_ctx = new_ctx(0.1, "carve")
    try:
        feed(src_ctx, runs["hdl64"], "carve")
        src = src_ctx.dense_snapshot()
        assert int(src["misses"].astype(bool).sum()) > 0
        # zero pose == no pose, both == the snapshot (resume)
        a, b = new_ctx(0.1, "map"), new_ctx(0.1, "map")
        try:
            a.dense_merge(src)
            b.dense_merge(src, np.zeros(6, np.float32))
            assert_snap(a.dense_snapshot(), src, "no pose")
            assert_snap(b.dense_snapshot(), src, "zero pose")
        finally:
            a.close()
            b.close()
        # the map merged into itself: counts and sums exactly doubled, evidence doubled with saturation
        self_ctx = new_ctx(0.1, "map")
        try:
            self_ctx.dense_merge(src)
            got, ref, _, _, _ = merge_both(self_ctx, 0.1, 2**31 - 1, src, None)
            assert_snap(got, ref.snapshot(), "into itself")
            assert np.array_equal(got["counts"], 2 * src["counts"])
            assert np.array_equal(got["sums"], 2.0 * src["sums"])
            assert np.array_equal(got["hits"], np.minimum(2 * src["hits"].astype(np.int64), 65535))
        finally:
            self_ctx.close()
        # under poses into another session's map, into a larger leaf, and past the key range; with a cap
        other = new_ctx(0.1, "map")
        try:
            feed(other, runs["vlp16"], "map")
            for twist in ((0.0, math.radians(5.0), 0.0, 0.8, 0.1, -0.6), (0.03, -2.0, -0.02, 12.5, -0.3, 7.75)):
                got, ref, went, s0, s1 = merge_both(other, 0.1, 2**31 - 1, src, twist)
                assert_snap(got, ref.snapshot(), f"pose {twist}")
                assert went["stored"] > 0 and went["new"] > 0
        finally:
            other.close()
        for leaf, twist in ((0.4, None), (0.2, (0.0, 1.0, 0.0, -3.0, 0.5, 2.0))):
            coarse = new_ctx(leaf, "map")
            try:
                got, ref, went, _, _ = merge_both(coarse, leaf, 2**31 - 1, src, twist)
                assert_snap(got, ref.snapshot(), f"into leaf {leaf}")
                assert got["keys"].size < src["keys"].size and int(got["counts"].sum()) == int(src["counts"].sum())
            finally:
                coarse.close()
        capped = new_ctx(0.1, "map", src["keys"].size // 2)
        try:
            got, ref, went, s0, s1 = merge_both(capped, 0.1, src["keys"].size // 2, src,
                                                (0.0, 0.0, 0.0, 2**20 * 0.1 - 20.0, 0.0, 0.0))
            assert_snap(got, ref.snapshot(), "cap and key range")
            assert went["skipped"] > 0 and went["dropped"] > 0
            assert s1["skipped"] - s0["skipped"] == went["skipped"] and s1["dropped"] - s0["dropped"] == went["dropped"]
        finally:
            capped.close()
    finally:
        src_ctx.close()


def test_two_sessions(build_libs, scene):
    """Session B's frame is its first sweep's pose, at an unknown heading a few metres off in session A's map.
    Relocalising B's first sweep in A's target gives that pose; B's snapshot merged under it lands where a merge under
    the true transform does."""
    from loam_velodyne_b200 import api, synth
    lidar, leaf = synth.Lidar.hdl64(1024), 0.2
    truth = np.array([0.01, 0.9, -0.01, 1.2, 0.0, 5.5], np.float32)  # B's origin in A's frame
    M = ar.to_map64(truth.astype(np.float64), np.eye(3))             # rows: images of the unit vectors
    A, _ = map_ctx(scene, lidar, leaf)
    B = new_ctx(leaf, "map")
    try:
        A.dense_target_build(None, 2)
        first = None
        for k in range(3):
            w_pose = truth.astype(np.float64) + np.array([0.0, 0.05 * k, 0.0, 0.3 * k, 0.0, 1.5 * k])
            sensor, world = ar.static_sweep(scene, lidar, w_pose, seed=300 + k)
            first = sensor if k == 0 else first
            in_b = (world[:, :3].astype(np.float64) - truth[3:].astype(np.float64)) @ M.T
            B.cloud_upload(api.C_MAP_FULL, np.concatenate([in_b.astype(np.float32), world[:, 3:]], axis=1))
            B.dense_insert(api.C_MAP_FULL)
        snap = B.dense_snapshot()
        a = 2.1
        prior = truth + np.array([0, -1.3, 0, 1.5 * math.cos(a), 0, 1.5 * math.sin(a)], np.float32)
        hyps = api.reloc_grid(prior, api.RELOC_YAW_STEP_DEG, None, api.RELOC_XZ_STEP, api.RELOC_XZ_STEPS)
        cands = A.dense_relocalize(first, hyps)
        assert cands
        est = cands[0]["fine"][0]
        e_m, e_deg = ar.twist_error(est, truth)
        assert e_m <= BAR_M and e_deg <= BAR_DEG, (e_m, e_deg)
        keys = {}
        for name, twist in (("estimate", est), ("truth", truth)):
            c = new_ctx(leaf, "map")
            try:
                c.dense_merge(snap, twist)
                keys[name] = c.dense_snapshot()["keys"]
            finally:
                c.close()
        share = np.intersect1d(keys["estimate"], keys["truth"]).size / keys["truth"].size
        before = A.dense_stats()["voxels"]
        A.dense_merge(snap, est)
        grown = A.dense_stats()["voxels"] - before
        print(f"pose error {e_m * 1000:.2f} mm {e_deg:.4f} deg; keys in common {share:.4f}; A grew by {grown} of "
              f"{snap['keys'].size} voxels")
        assert share >= SHARE_BAR
        assert 0 < grown < snap["keys"].size
    finally:
        A.close()
        B.close()


def test_mapping_stage_and_file(build_libs, scene, map_200k, tmp_path):
    """On the mapping stage's own map the drop-in snapshot and merge equal the Ctx path bit for bit; save -> load ->
    merge equals merging the snapshot in memory."""
    from loam_velodyne_b200 import api, synth
    from test_dense_align import SUMS
    reg = api.ScanRegistration()
    m = api.LaserMapping(0.1, 10)
    m.seed(*map_200k)
    m.enable_dense_map(0.1)
    lidar = synth.Lidar.vlp16(n_az=900)
    for it, sum6 in enumerate(SUMS[:6]):
        pts, rs = synth.make_sweep(scene, lidar, it, yaw_rate=math.radians(5.0))
        reg.process(pts, rs)
        m.set_inputs(reg.cloud("less_sharp"), reg.cloud("less_flat"), pts)
        m.update_odometry(np.asarray(sum6, np.float32))
        assert m.process()
    snap = m.dense_map_snapshot()
    cent, cnt = m.dense_map()
    assert snap["keys"].size == cnt.size > 1000 and np.array_equal(snap["counts"], cnt)
    assert np.array_equal((snap["sums"] / cnt[:, None].astype(np.float64)).astype(np.float32).view(np.uint32),
                          cent.view(np.uint32))
    twist = (0.0, 0.4, 0.0, 1.0, 0.0, -0.5)
    c = api.Ctx(0)
    try:
        c.dense_enable(0.1)
        c.dense_merge(snap)
        assert_snap(c.dense_snapshot(), snap, "Ctx resume")
        c.dense_merge(snap, twist)
        m.merge_dense_map(snap, twist)
        assert_snap(m.dense_map_snapshot(), c.dense_snapshot(), "drop-in merge")
        path = str(tmp_path / "map.npz")
        api.save_dense_snapshot(path, snap)
        back = api.load_dense_snapshot(path)
        assert back["leaf"] == np.float32(0.1)
        assert_snap(back, snap, "file")
        d = api.Ctx(0)
        try:
            d.dense_enable(0.1)
            d.dense_merge(back, twist)
            e = api.Ctx(0)
            try:
                e.dense_enable(0.1)
                e.dense_merge(snap, twist)
                assert_snap(d.dense_snapshot(), e.dense_snapshot(), "file merge")
            finally:
                e.close()
        finally:
            d.close()
    finally:
        c.close()


def test_lifecycle_errors_and_launches(build_libs, runs):
    """A merge leaves the target, its ray index and distance field alone; every refused call returns its code and
    changes nothing; launches are fixed per call, none for n == 0 or while the calls are unused."""
    from loam_velodyne_b200 import api
    import ctypes as C
    run = runs["vlp16"]
    c = new_ctx(0.2, "map")
    try:
        feed(c, run[:4], "map")
        c.dense_target_build(None, 2)
        pts, tw = run[5][0], run[5][1]
        rays = pts[::7]
        cast0 = c.dense_raycast(rays, tw)
        it0 = c.dense_align_iterate(pts, tw, 2)
        probe = np.array([[0.5, 0.5, 0.5, 0.0], [3.0, -1.0, 2.0, 0.0]], np.float32)
        dist0 = c.dense_distance_field((-20, -10, -20), (64, 32, 64), 2.0)
        q0 = c.dense_distance_query(probe, gradient=True)
        snap = c.dense_snapshot()
        c.dense_merge(snap, (0.0, 0.3, 0.0, 2.0, 0.0, 1.0))
        assert not np.array_equal(c.dense_snapshot()["counts"].sum(), snap["counts"].sum())
        cast1 = c.dense_raycast(rays, tw)
        it1 = c.dense_align_iterate(pts, tw, 2)
        assert all(np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
                   for x, y in zip(cast0, cast1))
        assert np.array_equal(it0[0]["AtA"], it1[0]["AtA"]) and it0[0]["n_selected"] == it1[0]["n_selected"]
        q1 = c.dense_distance_query(probe, gradient=True)
        assert np.all(np.isfinite(q0[0])) and dist0[0].shape == (64, 32, 64)
        assert all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(q0, q1))

        # errors: codes, and nothing changes
        state = c.dense_snapshot()
        arr = mr.entries([(1, 1, 0, 0.1, 0.1, 0.1, 1.0), (2, 3, 1, 0.3, 0.3, 0.3, 2.0)])
        L = c.L

        def raw_merge(s, pose=None, n=None, null=None):
            a = api._merge_arrays(s)
            ptrs = list(api._merge_ptrs(a))
            if n is not None:
                ptrs[4] = n
            if null is not None:
                ptrs[null] = None
            return L.loam_b200_dense_merge(c.h, *ptrs, C.byref(pose) if pose is not None else None)

        bad = []
        for field, i, value in (("counts", 1, 0), ("hits", 0, 0), ("sums", (1, 2), np.nan), ("sums", (0, 3), np.inf)):
            s = {k: np.array(v, copy=True) if v is not None else None for k, v in arr.items()}
            s[field][i] = value
            bad.append(raw_merge(s))
        bad.append(raw_merge(arr, api.make_pose((0.0, float("nan"), 0.0, 0.0, 0.0, 0.0))))
        bad.append(raw_merge(arr, api.make_pose((0.0, 0.0, 0.0, 0.0, float("inf"), 0.0))))
        bad.append(raw_merge(arr, n=-1))
        for null in range(4):
            bad.append(raw_merge(arr, null=null))
        assert bad == [-1] * len(bad), bad
        n = C.c_int(0)
        keys = np.zeros(4, np.uint64)
        assert L.loam_b200_dense_snapshot(c.h, keys.ctypes.data_as(C.POINTER(C.c_uint64)), None, None, None, None, 4,
                                          C.byref(n)) == -5 and n.value == state["keys"].size
        big = state["keys"].size
        assert L.loam_b200_dense_snapshot(c.h, None, None, None, None, None, big, C.byref(n)) == -1
        assert L.loam_b200_dense_snapshot(c.h, None, None, None, None, None, -1, C.byref(n)) == -1
        assert_snap(c.dense_snapshot(), state, "after the refused calls")
        empty = api.Ctx(0)
        try:
            assert empty.dense_snapshot()["keys"].size == 0
            with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
                empty.dense_merge(arr)
            empty.map_set_shard(0, 2)
            with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
                empty.dense_merge(arr)
        finally:
            empty.close()

        # launches: n == 0 launches nothing; a merge launches what an insertion of as many points does (no growth),
        # with carve mode on one more each; a snapshot what the export does
        c.cloud_upload(api.C_MAP_FULL, run[0][0][:5000])

        def launches(fn):
            c.dense_stats()
            before = c.launch_count()
            fn()
            c.dense_stats()
            return c.launch_count() - before

        few = {k: v[:5000] for k, v in state.items() if k != "leaf"}
        for _ in range(2):
            c.dense_merge(few)
            c.dense_insert(api.C_MAP_FULL)
        assert launches(lambda: c.dense_merge(mr.entries(np.zeros((0, 7))))) == 0
        ins = launches(lambda: c.dense_insert(api.C_MAP_FULL))
        mrg = launches(lambda: c.dense_merge(few))
        snp = launches(c.dense_snapshot)
        exp = launches(c.dense_export)
        assert mrg == ins and snp == exp, (mrg, ins, snp, exp)
        c.profile(True)
        c.dense_merge(few)
        c.dense_snapshot()
        prof = c.profile_get()
        assert sum(v[1] for k, v in prof.items() if k != "dense") == 0 and prof["dense"][1] == mrg + snp
        c.profile(False)
        c.dense_carving(0.5, 60.0)
        for _ in range(2):
            c.dense_merge(few)
            c.dense_insert(api.C_MAP_FULL)
        assert launches(lambda: c.dense_merge(few)) == launches(lambda: c.dense_insert(api.C_MAP_FULL)) == ins + 1
        print(f"launches: merge {mrg}, snapshot {snp}")
    finally:
        c.close()


def test_pipeline_in_flight(build_libs, scene):
    from loam_velodyne_b200 import api, synth
    lidar = synth.Lidar.vlp16()
    sweeps = [synth.make_sweep(scene, lidar, i, yaw_rate=math.radians(5.0)) for i in range(3)]
    pl = api.Pipeline()
    pl.mapping.enable_dense_map(0.1)
    pl.submit(*sweeps[0])
    while pl.collect(wait=True) is not None:
        pass
    snap = pl.mapping.dense_map_snapshot()
    assert snap["keys"].size > 1000
    for q, rs in sweeps[1:]:
        pl.submit(q, rs)
    with pytest.raises(api.LoamB200Error, match="in flight"):
        pl.mapping.dense_map_snapshot()
    with pytest.raises(api.LoamB200Error, match="in flight"):
        pl.mapping.merge_dense_map(snap)
    while pl.collect(wait=True) is not None:
        pass
    pl.mapping.merge_dense_map(snap, (0.0, 0.0, 0.0, 0.0, 0.0, 0.0))
    assert pl.mapping.dense_map_snapshot()["keys"].size >= snap["keys"].size
