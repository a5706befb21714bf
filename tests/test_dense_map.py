"""The whole-run voxel map on the GPU (csrc/densemap.cuh) against its numpy restatement (tests/dense_reference.py),
bit for bit: counts, fp32 centroids, order, skipped and dropped points.  Kernel-level inserts cover the key edges, both
sort paths and table growth; the mapping stage and the streaming pipeline cover the hook into the end of a sweep."""
import math

import numpy as np
import pytest

import dense_reference as dr

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def assert_same(got, ref, what=""):
    """(centroids, counts) and stats of the GPU equal the restatement's bit for bit."""
    (gc, gn), gs = got
    rc, rn = ref.export()
    assert gs == ref.stats(), f"{what}: stats {gs} vs {ref.stats()}"
    assert gc.shape == rc.shape, what
    assert np.array_equal(gn, rn), f"{what}: counts differ"
    assert np.array_equal(bits(gc), bits(rc)), f"{what}: {int((bits(gc) != bits(rc)).any(axis=1).sum())} centroids differ"


def gpu_run(clouds, leaf, max_voxels=2**31 - 1, check_each=False, ref=None):
    from loam_velodyne_b200 import api
    c = api.Ctx(0)
    try:
        c.dense_enable(leaf, max_voxels)
        for i, pts in enumerate(clouds):
            c.cloud_upload(api.C_MAP_FULL, pts)
            c.dense_insert(api.C_MAP_FULL)
            if check_each:
                ref.insert(pts)
                assert_same((c.dense_export(), c.dense_stats()), ref, f"insert {i}")
        return c.dense_export(), c.dense_stats()
    finally:
        c.close()


def ref_run(clouds, leaf, max_voxels=2**31 - 1):
    r = dr.DenseMapRef(leaf, max_voxels)
    for pts in clouds:
        r.insert(pts)
    return r


def registered(pts, yaw, t):
    c, s = np.float32(math.cos(yaw)), np.float32(math.sin(yaw))
    p = np.array(pts, np.float32, copy=True)
    x, z = p[:, 0].copy(), p[:, 2].copy()
    p[:, 0] = c * x + s * z + np.float32(t[0])
    p[:, 1] = p[:, 1] + np.float32(t[1])
    p[:, 2] = -s * x + c * z + np.float32(t[2])
    return p


def box_cloud(n, lo, hi, seed, leaf):
    """n points in a box, snapped so that many share a voxel; intensities spread over several decades."""
    rng = np.random.RandomState(seed)
    p = rng.uniform(lo, hi, (n, 3)).astype(np.float32)
    p = (np.round(p / (leaf * 0.25)) * (leaf * 0.25) + rng.uniform(-1e-3, 1e-3, (n, 3))).astype(np.float32)
    inten = (rng.uniform(0, 1, n) * 10.0 ** rng.randint(-3, 4, n)).astype(np.float32)
    return np.ascontiguousarray(np.concatenate([p, inten[:, None]], axis=1), np.float32)


@pytest.fixture(scope="module")
def hdl_sweeps(scene):
    from loam_velodyne_b200 import synth
    lidar = synth.Lidar.hdl64()
    out = []
    for i in range(20):
        pts, _ = synth.make_sweep(scene, lidar, i, yaw_rate=math.radians(5.0))
        out.append(registered(pts, 0.3 * i, (-40.0 + 4.1 * i, 0.2 * i, 25.0 - 3.3 * i)))
    return out


@pytest.mark.parametrize("leaf", [0.05, 0.1, 0.4])
def test_key_edges(build_libs, leaf):
    pts = dr.key_edge_cloud(leaf)
    assert_same(gpu_run([pts, pts[::-1].copy()], leaf), ref_run([pts, pts[::-1].copy()], leaf), "key edges")


def test_empty_and_single_point(build_libs):
    empty = np.zeros((0, 4), np.float32)
    got = gpu_run([empty], 0.1)
    assert got[0][0].shape == (0, 4) and got[1] == {"voxels": 0, "skipped": 0, "dropped": 0}
    one = np.array([[-3.14159, 2.71828, -0.05, 7.5]], np.float32)
    assert_same(gpu_run([empty, one, empty], 0.1), ref_run([one], 0.1), "one point")


def test_identical_points_beyond_one_cluster(build_libs):
    """131 073 copies of one point: a single run longer than the cluster sort holds (onesweep path)."""
    p = np.tile(np.array([[1.2345, -6.789, 10.5, 3.25]], np.float32), (131073, 1))
    p[::7, 3] = 0.1
    assert_same(gpu_run([p], 0.1), ref_run([p], 0.1), "identical points")


@pytest.mark.parametrize("n", [131071, 131072, 131073, 400000])
def test_both_sort_paths(build_libs, n):
    """Clouds up to 131 072 points sort in one cluster launch, larger ones through the onesweep passes."""
    clouds = [box_cloud(n, (-20, -3, -20), (20, 3, 20), 11, 0.2), box_cloud(n, (-5, -3, -5), (35, 3, 35), 12, 0.2)]
    assert_same(gpu_run(clouds, 0.2), ref_run(clouds, 0.2), f"n = {n}")


def test_hdl64_sweeps_with_table_growth(build_libs, hdl_sweeps):
    """20 registered HDL-64E sweeps at 0.05 m: the table grows (and rehashes) several times on the way."""
    ref = dr.DenseMapRef(0.05)
    got = gpu_run(hdl_sweeps, 0.05, check_each=False)
    for pts in hdl_sweeps:
        ref.insert(pts)
    first = dr.DenseMapRef(0.05)
    first.insert(hdl_sweeps[0])
    assert ref.stats()["voxels"] > 8 * first.stats()["voxels"]  # > 1024 -> 2^21+ slots: at least 3 rehashes
    assert_same(got, ref, "20 HDL-64E sweeps")


def test_fresh_runs_are_bit_identical(build_libs, hdl_sweeps):
    """The hash places entries wherever the CAS races put them; the export does not depend on it."""
    a = gpu_run(hdl_sweeps[:6], 0.05)
    b = gpu_run(hdl_sweeps[:6], 0.05)
    assert a[1] == b[1]
    assert np.array_equal(a[0][1], b[0][1]) and np.array_equal(bits(a[0][0]), bits(b[0][0]))


def order_cloud(n_vox, seed, leaf):
    """Voxels of 2-7 points whose intensities cancel catastrophically in fp64 (+-2^60, +-2^55 next to 1 and 3): the
    centroid depends on the order in which a voxel's points are summed.  The cloud is shuffled, so a voxel's points are
    spread over it."""
    rng = np.random.RandomState(seed)
    side = int(math.ceil(n_vox ** (1.0 / 3.0)))
    vox = np.stack(np.unravel_index(rng.choice(side ** 3, n_vox, replace=False), (side, side, side)), axis=1) - side // 2
    per = rng.randint(2, 8, n_vox)
    centre = np.repeat(vox, per, axis=0).astype(np.float32)
    p = ((centre + rng.uniform(0.1, 0.9, centre.shape)) * np.float32(leaf)).astype(np.float32)
    inten = rng.choice(np.float32([1.0, 3.0, 2.0 ** 60, -(2.0 ** 60), 2.0 ** 55, -(2.0 ** 55)]), p.shape[0])
    pts = np.concatenate([p, inten[:, None].astype(np.float32)], axis=1)
    return np.ascontiguousarray(pts[rng.permutation(pts.shape[0])], np.float32)


@pytest.mark.parametrize("n_vox", [20000, 60000])
def test_summation_order(build_libs, n_vox):
    """Within a sweep a voxel's points are summed in ascending cloud index, and sweeps add up in order.  The clouds here
    (~90 k and ~270 k points: both sort paths) change many centroids when that order is reversed."""
    leaf = 0.2
    clouds = [order_cloud(n_vox, 1, leaf), order_cloud(n_vox, 2, leaf)]
    ref = ref_run(clouds, leaf)
    rev = ref_run([c[::-1].copy() for c in clouds], leaf)
    assert np.count_nonzero(bits(ref.export()[0]) != bits(rev.export()[0])) > n_vox // 100
    assert_same(gpu_run(clouds, leaf), ref, "summation order")


def test_cap_mid_sweep(build_libs):
    """max_voxels is reached in the middle of the second cloud: its new voxels are admitted in ascending key order, the
    points of the rest are dropped, and voxels already stored keep accumulating in later clouds."""
    leaf = 0.2
    c1 = box_cloud(60000, (-10, -2, -10), (10, 2, 10), 1, leaf)
    c2 = box_cloud(60000, (0, -2, 0), (20, 2, 20), 2, leaf)
    c3 = box_cloud(60000, (-10, -2, -10), (20, 2, 20), 3, leaf)
    r1 = ref_run([c1], leaf)
    r12 = ref_run([c1, c2], leaf)
    v1, v12 = r1.stats()["voxels"], r12.stats()["voxels"]
    cap = v1 + (v12 - v1) // 2
    ref = dr.DenseMapRef(leaf, cap)
    got = gpu_run([c1, c2, c3], leaf, cap, check_each=True, ref=ref)
    s = got[1]
    assert s["voxels"] == cap and s["dropped"] > 0
    # the admitted voxels of the second cloud are the smallest new keys; the third cloud still adds to stored voxels
    r = dr.DenseMapRef(leaf, cap)
    r.insert(c1)
    r.insert(c2)
    new_keys = np.setdiff1d(r12.keys, r1.keys)
    assert np.array_equal(np.setdiff1d(r.keys, r1.keys), new_keys[:cap - v1])
    assert int(got[0][1].sum()) > int(r.count.sum())


SUMS = [(0.01, 1.3, -0.02, 0.3, 0.1, 0.2), (-0.02, 2.4, 0.03, 24.9, 0.5, 24.8), (0.0, -1.1, 0.0, -74.9, 0.2, -25.1),
        (0.03, 3.0, -0.01, -380.0, 1.0, 10.0), (0.0, -2.9, 0.02, 380.0, -1.0, -30.0), (0.0, 0.4, 0.0, -5.0, 0.0, 3.0)]
SUMS += [(0.0, 0.05 * i, 0.0, 0.4 * i, 0.02 * i, 0.9 * i) for i in range(16)]


def mapping_run(scene, map_200k, dense):
    """The mapping stage on its own (GPU scan registration for the features), seeded map, sums that roll the grid by
    +1 and -2 and sweeps far from the map (optimisation skipped).  -> per-sweep outputs, registered clouds, object."""
    from loam_velodyne_b200 import api, synth
    reg = api.ScanRegistration()
    m = api.LaserMapping(0.1, 10)
    m.seed(*map_200k)
    if dense:
        m.enable_dense_map(0.1)
    lidar = synth.Lidar.vlp16(n_az=900)
    outs, fulls = [], []
    for it, sum6 in enumerate(SUMS):
        pts, rs = synth.make_sweep(scene, lidar, it, yaw_rate=math.radians(5.0))
        reg.process(pts, rs)
        m.set_inputs(reg.cloud("less_sharp"), reg.cloud("less_flat"), pts)
        m.update_odometry(np.asarray(sum6, np.float32))
        assert m.process()
        full = m.cloud("full")
        fulls.append(full)
        outs.append((m.twist("aft"), m.twist("bef"), m.twist("tobe"), full, m.cloud("surf_stack_ds")))
    outs.append((m.cloud("corner_cubes"), m.cloud("surf_cubes")))
    return outs, fulls, m


def test_mapping_stage(build_libs, scene, map_200k):
    off, _, _ = mapping_run(scene, map_200k, False)
    on, fulls, m = mapping_run(scene, map_200k, True)
    for i, (a, b) in enumerate(zip(off, on)):
        for x, y in zip(a, b):
            assert np.array_equal(bits(x), bits(y)), f"sweep {i}: an output changed with the whole-run map on"
    ref = ref_run(fulls, 0.1)
    assert ref.stats()["voxels"] > 10000
    assert_same((m.dense_map(), m.dense_stats()), ref, "mapping stage")
    m.clear_dense_map()
    assert m.dense_stats() == {"voxels": 0, "skipped": 0, "dropped": 0}


def test_streaming_pipeline(build_libs, scene, map_200k):
    from loam_velodyne_b200 import api, synth
    lidar = synth.Lidar.vlp16()
    sweeps = [synth.make_sweep(scene, lidar, i, yaw_rate=math.radians(5.0)) for i in range(12)]
    seq = api.Pipeline()
    seq.seed_map(*map_200k)
    seq.mapping.enable_dense_map(0.1)
    res_seq = [seq.sweep(p, rs) for p, rs in sweeps]
    st = api.Pipeline()
    st.seed_map(*map_200k)
    st.mapping.enable_dense_map(0.1)
    res_st = st.run_stream(sweeps)
    for a, b in zip(res_seq, res_st):
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    a, b = seq.mapping.dense_map(), st.mapping.dense_map()
    assert seq.mapping.dense_stats() == st.mapping.dense_stats()
    assert a[0].shape[0] > 10000
    assert np.array_equal(a[1], b[1]) and np.array_equal(bits(a[0]), bits(b[0]))


def test_errors(build_libs, scene):
    from loam_velodyne_b200 import api, synth
    c = api.Ctx(0)
    for leaf, cap in ((0.0, 10), (-0.1, 10), (float("nan"), 10), (float("inf"), 10), (0.1, 0), (0.1, 2**31)):
        with pytest.raises(api.LoamB200Error, match="invalid argument"):
            c.dense_enable(leaf, cap)
    with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
        c.dense_insert(api.C_MAP_FULL)  # not enabled
    c.dense_enable(0.1)
    c.dense_enable(0.2)  # empty map: the leaf may change
    c.cloud_upload(api.C_MAP_FULL, np.array([[1, 2, 3, 4]], np.float32))
    c.dense_insert(api.C_MAP_FULL)
    c.dense_enable(0.2, 5)  # same leaf: the cap may change
    with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
        c.dense_enable(0.1)
    c.dense_clear()
    c.dense_enable(0.1)
    c.close()
    s = api.Ctx(0)
    s.map_set_shard(0, 2)
    with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
        s.dense_enable(0.1)
    s.close()
    m = api.LaserMapping()
    m.enable_sharding(1, 2, None)
    with pytest.raises(api.LoamB200Error, match="invalid call sequence"):
        m.enable_dense_map(0.1)
    # a sweep is in flight from submit() until its result is collected: refused before the results are taken (whatever
    # the stages have finished meanwhile), allowed once every result has been collected
    lidar = synth.Lidar.vlp16()
    sweeps = [synth.make_sweep(scene, lidar, i, yaw_rate=math.radians(5.0)) for i in range(4)]
    p = api.Pipeline()
    p.mapping.enable_dense_map(0.1)
    for pts, rs in sweeps:
        p.submit(pts, rs)
    for k in range(len(sweeps)):
        for call in (p.mapping.dense_map, p.mapping.dense_stats, p.mapping.clear_dense_map):
            with pytest.raises(api.LoamB200Error, match="in flight"):
                call()
        assert p.collect(wait=True) is not None
    assert p.collect(wait=True) is None
    pts, n = p.mapping.dense_map()
    assert pts.shape[0] == p.mapping.dense_stats()["voxels"] > 0
    p.sync()
    assert np.array_equal(p.mapping.dense_map()[1], n)


def test_cap_lowered_below_stored_voxels(build_libs):
    """Enabling again with the same leaf changes the cap.  A cap below the stored voxels keeps them (they go on
    accumulating) and admits no new voxel; raising it again admits new voxels in key order up to the new cap."""
    from loam_velodyne_b200 import api
    leaf = 0.2
    c1 = box_cloud(50000, (-10, -2, -10), (10, 2, 10), 21, leaf)
    c2 = box_cloud(50000, (-5, -2, -5), (15, 2, 15), 22, leaf)
    c3 = box_cloud(50000, (0, -2, 0), (20, 2, 20), 23, leaf)
    ref = dr.DenseMapRef(leaf)
    c = api.Ctx(0)
    try:
        c.dense_enable(leaf)
        ref.insert(c1)
        v1 = ref.stats()["voxels"]
        steps = [(v1 // 2, c2), (v1 // 2, c1), (v1 + 3000, c3)]
        c.cloud_upload(api.C_MAP_FULL, c1)
        c.dense_insert(api.C_MAP_FULL)
        assert_same((c.dense_export(), c.dense_stats()), ref, "before the cap")
        for i, (cap, pts) in enumerate(steps):
            c.dense_enable(leaf, cap)
            ref.max_voxels = cap
            c.cloud_upload(api.C_MAP_FULL, pts)
            c.dense_insert(api.C_MAP_FULL)
            ref.insert(pts)
            assert_same((c.dense_export(), c.dense_stats()), ref, f"cap {cap}, insert {i}")
        s = c.dense_stats()
        assert s["voxels"] == v1 + 3000 and s["dropped"] > 0
    finally:
        c.close()
