"""The numpy restatement of the whole-run map's normals (tests/normals_reference.py) on the CPU: its vectorised sums
against a plain per-voxel loop, its fp32 eigenvectors against float64, analytic surfaces, and the hand-made edge cases
each shown to catch a deliberately wrong restatement."""
import math

import numpy as np
import pytest

import dense_reference as dr
import normals_reference as nr

EPS32 = float(np.finfo(np.float32).eps)
# fp32 normals against the float64 eigenvector of the same neighbourhood: sin(angle) <= C_BAR * eps32 * |C| / gap.
# The covariance is rounded to fp32 entry by entry (a perturbation of about eps32 * |C|) and the solver works in fp32;
# the worst of the 34 k fits below is 4.4 (printed).
C_BAR = 16.0


@pytest.fixture(scope="module")
def drv(build_libs):
    from oracle import pydriver
    return pydriver.best()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def export(pts, leaf):
    r = dr.DenseMapRef(leaf)
    r.insert(pts)
    return r.keys, r.export()[0]


def box_cloud(n, lo, hi, seed, leaf):
    rng = np.random.RandomState(seed)
    p = rng.uniform(lo, hi, (n, 3)).astype(np.float32)
    p = (np.round(p / (leaf * 0.25)) * (leaf * 0.25) + rng.uniform(-1e-3, 1e-3, (n, 3))).astype(np.float32)
    return np.ascontiguousarray(np.concatenate([p, np.ones((n, 1), np.float32)], axis=1), np.float32)


def plane_cloud(normal, origin, half, n, seed):
    """n points uniformly on a square patch (side 2 * half) of the plane through `origin` with `normal`."""
    rng = np.random.RandomState(seed)
    nrm = np.asarray(normal, np.float64) / np.linalg.norm(normal)
    e1 = np.cross(nrm, [0.0, 0.0, 1.0] if abs(nrm[2]) < 0.9 else [1.0, 0.0, 0.0])
    e1 /= np.linalg.norm(e1)
    e2 = np.cross(nrm, e1)
    uv = rng.uniform(-half, half, (n, 2))
    p = np.asarray(origin, np.float64) + uv[:, :1] * e1 + uv[:, 1:] * e2
    return np.concatenate([p, np.ones((n, 1))], axis=1).astype(np.float32), nrm, e1, e2


def sphere_cloud(centre, radius, n, seed):
    rng = np.random.RandomState(seed)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    p = np.asarray(centre, np.float64) + radius * d
    return np.concatenate([p, np.ones((n, 1))], axis=1).astype(np.float32)


@pytest.mark.parametrize("radius", [1, 2, 3])
def test_vectorised_equals_loop(drv, radius):
    """A few thousand voxels of mixed density (sparse corners give k < 3), two viewpoints: bit for bit, NaN alike."""
    leaf = 0.1
    pts = np.concatenate([box_cloud(6000, (-0.8, -0.4, -0.8), (0.8, 0.4, 0.8), 1, leaf),
                          box_cloud(40, (2, 2, 2), (4, 4, 4), 2, leaf)])
    keys, cent = export(pts, leaf)
    if radius == 3:  # the loop visits 343 offsets per voxel
        keys, cent = keys[::4].copy(), cent[::4].copy()
    assert keys.size > (300 if radius == 3 else 2000)
    for vp in ((0.0, 0.0, 0.0), (13.7, -250.0, 3.3)):
        a = nr.normals(keys, cent, radius, vp, drv)
        b = nr.normals_loop(keys, cent, radius, vp, drv)
        assert np.isnan(a[:, 0]).any() and (~np.isnan(a[:, 0])).sum() > keys.size // 2
        assert np.array_equal(bits(a), bits(b))


def test_against_float64(drv):
    """fp32 normals against numpy's float64 eigh of the unrounded covariance of the same neighbourhoods."""
    worst = 0.0
    fits = 0
    for leaf, pts in ((0.1, box_cloud(20000, (-1.5, -0.5, -1.5), (1.5, 0.5, 1.5), 3, 0.1)),
                      (0.05, plane_cloud((0.3, 1.0, 0.2), (2.0, -1.0, 4.0), 1.0, 60000, 4)[0]),
                      (0.1, sphere_cloud((1.0, -2.0, 0.5), 2.0, 80000, 5))):
        keys, cent = export(pts, leaf)
        for radius in (1, 2):
            S1, S2, k = nr.sums(keys, cent, radius)
            got = nr.normals(keys, cent, radius, (0.0, 0.0, 0.0), drv)
            for i in np.nonzero(k >= 3)[0]:
                kd = float(k[i])
                C = np.empty((3, 3))
                for j, (a, b) in enumerate(((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))):
                    C[a, b] = C[b, a] = (S2[i, j] - S1[i, a] * S1[i, b] / kd) / kd
                ev, V = np.linalg.eigh(C)
                gap = ev[1] - ev[0]
                if not gap > 0.0:
                    continue
                n = got[i, :3].astype(np.float64)
                sin = np.linalg.norm(np.cross(n / np.linalg.norm(n), V[:, 0]))
                worst = max(worst, sin / (EPS32 * np.abs(ev).max() / gap))
                fits += 1
    print(f"{fits} fits, worst sin(angle) = {worst:.3f} * eps32 * |C| / gap")
    assert fits > 10000
    assert worst <= C_BAR


@pytest.mark.parametrize("leaf", [0.05, 0.1, 0.4])
def test_tilted_planes(drv, leaf):
    """Centroids of coplanar points are coplanar: interior normals within 0.01 deg of the plane's, curvature ~0."""
    pts, nrm, e1, e2 = plane_cloud((0.3, 1.0, -0.45), (3.0, -1.5, 7.0), 40 * leaf, 200000, 6)
    keys, cent = export(pts, leaf)
    for radius in (1, 2, 3):
        got = nr.normals(keys, cent, radius, (0.0, 50.0, 0.0), drv)
        rel = cent[:, :3].astype(np.float64) - (3.0, -1.5, 7.0)
        inner = (np.abs(rel @ e1) < 40 * leaf - 2 * (radius + 1) * leaf) & (np.abs(rel @ e2) < 40 * leaf - 2 * (radius + 1) * leaf)
        assert inner.sum() > 500
        n = got[inner, :3].astype(np.float64)
        n /= np.linalg.norm(n, axis=1, keepdims=True)
        ang = np.degrees(np.arcsin(np.minimum(np.linalg.norm(np.cross(n, nrm), axis=1), 1.0)))
        assert np.all(ang < 0.01), f"radius {radius}: {ang.max()} deg"
        assert np.all(np.abs(got[inner, 3]) < 1e-5)


def test_sphere(drv):
    """Normals of a 2 m sphere at 0.1 m are radial; they point outward where an outside viewpoint sees the surface and
    inward everywhere from the centre."""
    centre = np.array([1.0, -2.0, 0.5])
    keys, cent = export(sphere_cloud(centre, 2.0, 300000, 8), 0.1)
    c = cent[:, :3].astype(np.float64)
    radial = (c - centre) / np.linalg.norm(c - centre, axis=1, keepdims=True)
    outside = centre + (0.0, 0.0, 30.0)
    for radius in (1, 2):
        got = nr.normals(keys, cent, radius, outside, drv)
        ok = ~np.isnan(got[:, 0])
        n = got[:, :3].astype(np.float64)
        ang = np.degrees(np.arccos(np.clip(np.abs(np.einsum("ij,ij->i", n, radial)), 0, 1)))
        print(f"radius {radius}: radial within {np.median(ang[ok]):.2f} deg (median), {ang[ok].max():.2f} deg (max)")
        assert ok.mean() > 0.99 and np.median(ang[ok]) < 1.0 and ang[ok].max() < 5.0
        to_vp = outside - c
        seen = ok & (np.einsum("ij,ij->i", radial, to_vp / np.linalg.norm(to_vp, axis=1, keepdims=True)) > 0.2)
        assert seen.sum() > 1000 and np.all(np.einsum("ij,ij->i", n[seen], radial[seen]) > 0)
        got = nr.normals(keys, cent, radius, centre, drv)
        ok = ~np.isnan(got[:, 0])
        assert np.all(np.einsum("ij,ij->i", got[ok, :3].astype(np.float64), radial[ok]) < 0)


@pytest.mark.parametrize("name", list(nr.edge_cases()))
def test_edge_cases_are_sensitive(drv, name):
    """Every hand-made case matches the per-voxel loop and changes under the wrong restatement it is built for: key
    arithmetic that wraps, a threshold of k < 2, a flip on <=.  (On the empty map nothing can differ.)"""
    pts, vp, variants = nr.edge_cases()[name]
    keys, cent = export(pts, nr.EDGE_LEAF)
    for radius in (1, 2, 3):
        right = nr.normals(keys, cent, radius, vp, drv)
        assert np.array_equal(bits(right), bits(nr.normals_loop(keys, cent, radius, vp, drv)))
    right = nr.normals(keys, cent, 1, vp, drv)
    if variants is None:
        assert keys.size == 0 and right.shape == (0, 4)
        return
    for v in variants if isinstance(variants, list) else [variants]:
        wrong = nr.normals(keys, cent, 1, vp, drv, **v)
        assert not np.array_equal(bits(right), bits(wrong)), f"{name}: {sorted(v)} gives the same answer"


def test_filtered_voxels_are_no_neighbours(drv):
    """Leaving a voxel out of the export changes its neighbours' normals: the restatement over the kept voxels differs
    from the one over every voxel restricted to the kept ones (which is what including filtered voxels would give)."""
    keys, cent = export(box_cloud(8000, (-1, -0.3, -1), (1, 0.3, 1), 9, 0.1), 0.1)
    kept = np.arange(keys.size) % 7 != 3
    right = nr.normals(keys[kept], cent[kept], 1, (0.0, 0.0, 0.0), drv)
    wrong = nr.normals(keys, cent, 1, (0.0, 0.0, 0.0), drv)[kept]
    differ = (bits(right) != bits(wrong)).any(axis=1)
    assert differ.sum() > keys.size // 4
