"""The shared radix sort, the voxel grid filter and the mapping stage's stack downsample on every launch path, bit for
bit against the plain restatements of tests/voxel_reference.py (pinned to the checker by test_voxel_reference.py).

Paths: the one-cluster sort and voxel filter (0 < n <= 131072 and clusters usable), onesweep with 4 items per thread
(n < 200000) or 16, and the multi-launch voxel grid above 131072 points or on a LOAM_B200_NO_CLUSTER=1 context.  Every
case runs on a default context and on a NO_CLUSTER one, and checks through debug_sort_pairs which path ran."""
import contextlib
import math
import os

import numpy as np
import pytest

import dense_reference as dr
import map_reference as mr
import voxel_reference as vr

pytestmark = pytest.mark.gpu

F = np.float32
CS_MAX_N = 131072
CTX_KINDS = ["cluster", "no_cluster"]


def _ctx(no_cluster=False):
    from loam_velodyne_b200 import api
    old = os.environ.get("LOAM_B200_NO_CLUSTER")
    if no_cluster:
        os.environ["LOAM_B200_NO_CLUSTER"] = "1"
    try:
        return api.Ctx(0)
    finally:
        if no_cluster:
            if old is None:
                del os.environ["LOAM_B200_NO_CLUSTER"]
            else:
                os.environ["LOAM_B200_NO_CLUSTER"] = old


@contextlib.contextmanager
def _closing(c):
    try:
        yield c
    finally:
        c.close()


@pytest.fixture(scope="module", params=CTX_KINDS)
def sctx(request):
    c = _ctx(no_cluster=request.param == "no_cluster")
    c.kind = request.param
    yield c
    c.close()


def expected_path(kind, n):
    if n <= 0:
        return -1
    if kind == "cluster" and n <= CS_MAX_N:
        return 0
    return 1 if n < 200000 else 2


def assert_path(c, n):
    """The path the sort (and the voxel grid, which makes the same choice) takes at n on this context."""
    _, _, path = c.debug_sort_pairs(np.zeros(n, np.uint32), np.zeros(n, np.int32), 32)
    assert path == expected_path(c.kind, n), f"n={n}: path {path}"


def bits(a):
    return np.ascontiguousarray(a, F).view(np.uint32)


# ---------------------------------------------------------------------------------------------------------- sort
SORT_SIZES = [1, 2, 31, 32, 33, 1023, 1024, 1025, 4095, 4096, 4097, 131071, 131072, 131073, 199999, 200000, 200001,
              2**22 + 5]
KEY_KINDS = ["uniform", "equal", "top_const", "low_const", "two_values", "many_ff", "ascending", "descending"]


def make_keys(kind, n, rng):
    u = rng.randint(0, 2**32, n, dtype=np.uint64).astype(np.uint32)
    if kind == "uniform":
        return u
    if kind == "equal":
        return np.full(n, 0x5A3C96E1, np.uint32)  # every pass skipped
    if kind == "top_const":
        return (u & np.uint32(0x00FFFFFF)) | np.uint32(0xA7000000)
    if kind == "low_const":
        return (u & np.uint32(0xFFFF00FF)) | np.uint32(0x0000002B)  # a skipped pass below two sorted ones
    if kind == "two_values":
        return np.where(u & np.uint32(1), np.uint32(0x80000001), np.uint32(0x7FFFFFFF)).astype(np.uint32)
    if kind == "many_ff":
        return np.where(u % np.uint32(3) == 0, u, np.uint32(0xFFFFFFFF)).astype(np.uint32)  # onesweep's pad key
    if kind == "ascending":
        return np.sort(u)
    return np.sort(u)[::-1].copy()


def check_sort(c, keys, key_bits=32, live=None, out_params=True):
    rng = np.random.RandomState(keys.shape[0] % 1000)
    vals = rng.randint(-2**31, 2**31, keys.shape[0], dtype=np.int64).astype(np.int32)
    gk, gv, path = c.debug_sort_pairs(keys, vals, key_bits, live=live, out_params=out_params)
    n = keys.shape[0]
    m = n if live is None else min(n, live)
    rk, rv = vr.sort_pairs(keys[:m], vals[:m], key_bits, out_params)
    assert np.array_equal(gk[:m], rk), f"keys differ at {np.flatnonzero(gk[:m] != rk)[:5]}"
    assert np.array_equal(gv[:m], rv), f"values differ at {np.flatnonzero(gv[:m] != rv)[:5]}"
    assert path == expected_path(c.kind, n), f"n={n}: path {path}"


@pytest.mark.parametrize("n", SORT_SIZES)
def test_sort_key_kinds(sctx, n):
    rng = np.random.RandomState(n % 7919)
    for kind in KEY_KINDS:
        check_sort(sctx, make_keys(kind, n, rng))


@pytest.mark.parametrize("n", [33, 4097, 131072, 131073, 200001])
def test_sort_key_bits_and_out_params(sctx, n):
    """Passes = ceil(key_bits / 8), rounded up to even for callers that read the first buffer: only those bits order
    the keys; the rest keep input order."""
    keys = make_keys("uniform", n, np.random.RandomState(n))
    for key_bits in (8, 16, 24, 30, 32):
        for out_params in (True, False):
            check_sort(sctx, keys, key_bits, out_params=out_params)


@pytest.mark.parametrize("live,n", [(0, 1000), (1000, 131072), (131072, 131073), (199999, 500000), (5000, 3000)])
def test_sort_live_count_on_device(sctx, live, n):
    keys = make_keys("uniform", n, np.random.RandomState(live))
    for key_bits, out_params in ((32, True), (8, True), (30, False)):
        check_sort(sctx, keys, key_bits, live=live, out_params=out_params)


def test_sort_arguments(sctx):
    import ctypes as C
    from loam_velodyne_b200 import api
    k = np.zeros(4, np.uint32)
    v = np.zeros(4, np.int32)
    for key_bits in (0, 33, -8):
        with pytest.raises(api.LoamB200Error, match="invalid argument"):
            sctx.debug_sort_pairs(k, v, key_bits)
    L, U, I = sctx.L, C.POINTER(C.c_uint32), C.POINTER(C.c_int)
    path = C.c_int(7)
    up, ip = k.ctypes.data_as(U), v.ctypes.data_as(I)
    assert L.loam_b200_debug_sort_pairs(sctx.h, up, ip, -1, -1, 32, 1, up, ip, C.byref(path)) == -1
    for i in range(5):
        a = [up, ip, up, ip, C.byref(path)]
        a[i] = None
        assert L.loam_b200_debug_sort_pairs(sctx.h, a[0], a[1], 4, -1, 32, 1, a[2], a[3], a[4]) == -1
    assert L.loam_b200_debug_sort_pairs(None, up, ip, 4, -1, 32, 1, up, ip, C.byref(path)) == -1
    gk, gv, p = sctx.debug_sort_pairs(np.zeros(0, np.uint32), np.zeros(0, np.int32), 32)
    assert gk.shape == (0,) and gv.shape == (0,) and p == -1


# ---------------------------------------------------------------------------------------------------- voxel grid
def check_voxel_grid(c, pts, leaf):
    pts = np.ascontiguousarray(pts, F)
    g = c.voxel_grid(pts, leaf)
    r = vr.voxel_grid(pts, leaf)
    assert g.shape == r.shape, f"{g.shape} vs {r.shape}"
    diff = np.flatnonzero(np.any(bits(g) != bits(r), axis=1))
    assert diff.size == 0, f"{diff.size} rows differ, first {diff[:5]}: {g[diff[:2]]} vs {r[diff[:2]]}"
    if pts.shape[0]:
        assert_path(c, pts.shape[0])
    return r


def moved(pts, yaw, t):
    c, s = F(math.cos(yaw)), F(math.sin(yaw))
    p = np.array(pts, F, copy=True)
    x, z = p[:, 0].copy(), p[:, 2].copy()
    p[:, 0] = c * x + s * z + F(t[0])
    p[:, 1] = p[:, 1] + F(t[1])
    p[:, 2] = -s * x + c * z + F(t[2])
    return p


@pytest.fixture(scope="module")
def sweeps(scene):
    from loam_velodyne_b200 import synth
    out = {}
    for name in ("vlp16", "hdl64", "dense128"):
        pts, _ = synth.make_sweep(scene, getattr(synth.Lidar, name)(), 3, yaw_rate=math.radians(5.0))
        out[name] = moved(pts, -2.1, (-131.3, -4.2, -57.9))
    out["hdl64_plus1"] = np.concatenate([out["hdl64"], out["hdl64"][17:18] + F(0.01)])
    assert [out[k].shape[0] for k in ("vlp16", "hdl64", "hdl64_plus1", "dense128")] == [28800, 131072, 131073, 524288]
    return out


@pytest.mark.parametrize("leaf", [0.05, 0.2, 0.4, 1.0])
@pytest.mark.parametrize("name", ["vlp16", "hdl64", "hdl64_plus1", "dense128"])
def test_voxel_grid_sweeps(sctx, sweeps, name, leaf):
    r = check_voxel_grid(sctx, sweeps[name], leaf)
    overflow = vr.voxel_meta(sweeps[name], leaf)[3]
    assert overflow == (leaf == 0.05 and name in ("vlp16", "dense128"))  # the widest sweeps trip the guard at 5 cm
    assert (r.shape[0] == sweeps[name].shape[0]) == overflow  # the input unchanged


@pytest.mark.parametrize("leaf", [0.05, 0.2, 0.4, 1.0])
def test_voxel_grid_key_edges(sctx, leaf):
    pts = dr.key_edge_cloud(leaf)
    check_voxel_grid(sctx, pts[np.all(np.abs(pts[:, :3]) < 100.0, axis=1)], leaf)


@pytest.mark.parametrize("n_background", [2000, 100000, 150000])
def test_voxel_grid_order_probes(sctx, n_background):
    """Runs whose float32 sums depend on the order: only input order within a voxel passes."""
    check_voxel_grid(sctx, vr.order_probe_cloud(n_background, seed=n_background), 1.0)


@pytest.mark.parametrize("n", [CS_MAX_N, CS_MAX_N + 1, 300000])
def test_voxel_grid_one_voxel(sctx, n):
    """One run across every CTA's shared memory of the cluster, and across many scan blocks."""
    rng = np.random.RandomState(n)
    frac = rng.uniform(0.0, 0.999, (n, 4)).astype(F)
    frac[rng.rand(n) < 0.5] *= F(1e-3)
    pts = frac + np.array([-3.0, 7.0, 12.0, 0.0], F)
    r = check_voxel_grid(sctx, pts, 1.0)
    assert r.shape[0] == 1


@pytest.mark.parametrize("n", [4096, 140000])
@pytest.mark.parametrize("box", list(vr.GUARD_BOXES))
def test_voxel_grid_guard_edges(sctx, box, n):
    pts = vr.guard_box_cloud(box, n=n, seed=n)
    r = check_voxel_grid(sctx, pts, 1.0)
    assert (r.shape[0] == n) == (box == "over")


def test_voxel_grid_tiny(sctx):
    assert sctx.voxel_grid(np.zeros((0, 4), F), 0.2).shape == (0, 4)
    one = np.array([[-1.25, 3.5, 0.1, 9.0]], F)
    check_voxel_grid(sctx, one, 0.2)
    check_voxel_grid(sctx, np.array([[0.01, 0.02, 0.03, 1.0], [0.07, 0.11, 0.13, 2.0]], F), 0.2)  # one voxel
    check_voxel_grid(sctx, np.array([[0.01, 0.02, 0.03, 1.0], [-0.07, 0.11, 0.13, 2.0]], F), 0.2)  # two


# -------------------------------------------------------------------------------------- stack downsample (mapping)
POSES = {  # zero rotation, and the poses of test_map_stage.py
    "zero": (0.0, 0.0, 0.0, 0.0, 0.0, 0.0),
    "cube_corner": (0.0, 0.0, 0.0, 24.5, 0.0, 24.5),
    "x_minus_75": (0.0, 0.0, 0.0, -74.5, 0.0, -20.5),
    "yaw": (0.01, 1.3, -0.02, 3.0, 0.2, 5.0),
}
LEAVES = (0.2, 0.4)


@pytest.fixture(scope="module")
def stacks(oracle, scene):
    """(corner, surface) stacks: a VLP-16 sweep's less-sharp / less-flat points; 131 072 / 131 073 points; a dense128
    sweep; and the VLP-16 stacks with two points at +-4000 m in the surface stack (the guard trips at 0.4 m)."""
    from loam_velodyne_b200 import synth
    s = oracle.scanreg()
    pts, rs = synth.make_sweep(scene, synth.Lidar.vlp16(), 3, yaw_rate=math.radians(5.0))
    s.process(pts, rs)
    ls, lf = s.cloud("less_sharp"), s.cloud("less_flat")
    hdl, _ = synth.make_sweep(scene, synth.Lidar.hdl64(), 2, yaw_rate=math.radians(5.0))
    dense, _ = synth.make_sweep(scene, synth.Lidar.dense128(), 1, yaw_rate=math.radians(5.0))
    far = np.array([[-4000.0, -4000.0, -4000.0, 1.0], [4000.0, 4000.0, 4000.0, 2.0]], F)
    return {
        "vlp16": (ls, lf),
        "131072_131073": (hdl, np.concatenate([hdl, hdl[5:6] + F(0.01)])),
        "dense128": (dense, lf),
        "far": (ls, np.concatenate([lf[:100], far, lf[100:]])),
    }


@pytest.mark.parametrize("pose_name", list(POSES))
@pytest.mark.parametrize("stack_name", ["vlp16", "131072_131073", "dense128", "far"])
@pytest.mark.parametrize("kind", CTX_KINDS)
def test_stack_downsample_as_the_pipeline_runs_it(map_200k, stacks, kind, stack_name, pose_name):
    from loam_velodyne_b200 import api
    twist = np.asarray(POSES[pose_name], F)
    corner, surf = stacks[stack_name]
    with _closing(_ctx(no_cluster=kind == "no_cluster")) as c:
        c.kind = kind
        for k in (0, 1):
            c.map_pool_append(k, map_200k[k])
        cen, valid, _ = mr.window(twist, (10, 5, 10))
        c.cloud_upload(api.C_MAP_CORNER_LAST, corner)
        c.cloud_upload(api.C_MAP_SURF_LAST, surf)
        sizes = c.map_begin_sweep(twist, cen, valid, *LEAVES)
        got = (c.cloud_download(api.C_MAP_CORNER_STACK_DS), c.cloud_download(api.C_MAP_SURF_STACK_DS))
        for i, (last, leaf) in enumerate(((corner, LEAVES[0]), (surf, LEAVES[1]))):
            rt = vr.stack_roundtrip(last, twist)
            ref = vr.voxel_grid(rt, leaf)
            assert sizes[2 + i] == ref.shape[0] == got[i].shape[0]
            diff = np.flatnonzero(np.any(bits(got[i]) != bits(ref), axis=1))
            assert diff.size == 0, f"stack {i}: {diff.size} rows differ, first {diff[:5]}"
            if stack_name == "far" and i == 1:
                assert np.array_equal(bits(got[i]), bits(rt))  # the round trip alone, apart from the filter
            assert_path(c, last.shape[0])
