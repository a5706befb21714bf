"""The plain reference of the scan-to-scan correspondence search (tests/odom_reference.py) against the checker's
restatement (oracle/loam_oracle.cpp, pinned to the compiled reference over whole streams by test_oracle.py), one
search iteration at zero twist.  The indices must agree bit for bit: the closest point up to an exact fp32 distance
tie (the k-d tree and the brute force may pick different members of a tie), the second and third points from the
checker's own closest point exactly, tie choices of the scans included.  The GPU stage tests (test_odom_stage.py)
then trust this reference without slack."""
import math

import numpy as np
import pytest

import odom_reference as orf

LIDARS = {"vlp16": 0, "hdl64": 2}


@pytest.fixture(scope="module")
def clouds(oracle, scene):
    from loam_velodyne_b200 import synth
    return {name: orf.last_and_current(oracle, getattr(synth.Lidar, name)(), sweep, scene, 5.0)
            for name, sweep in LIDARS.items()}


def _against_checker(oracle, lc, ls, sharp, flat, what, dense=True):
    from oracle import pydriver
    assert sharp.shape[0] <= lc.shape[0] and flat.shape[0] <= ls.shape[0]  # the checker reads past the end otherwise
    ref = pydriver.OdomIterator(oracle, lc, ls, sharp, flat).iterate(0, np.zeros(6, np.float32))["ind"]
    s = orf.Search(lc, ls)
    res = s.run(sharp, flat)
    ind = res["ind"]
    if dense:
        assert (ind[:, 0] >= 0).mean() > 0.8, f"{what}: few queries found a closest point"
        assert (ind[:, 1] >= 0).sum() > 50, what
    ns = sharp.shape[0]
    for k in np.flatnonzero((ind != ref).any(axis=1)):
        corner = k < ns
        assert ref[k, 0] in set(res["ties"][k].tolist()), f"{what}: query {k}: closest {ref[k]} vs {ind[k]}"
        last = lc if corner else ls
        d = orf.sq_dist(last, res["xyz"][k])
        got = orf.scans_from(last, d, int(ref[k, 0]), ns if corner else flat.shape[0], corner)
        assert got == (int(ref[k, 1]), int(ref[k, 2])), f"{what}: query {k}: scans from {ref[k, 0]}: {got} vs {ref[k]}"
    return res


@pytest.mark.parametrize("lidar", list(LIDARS))
def test_reference_search_ring_ordered(oracle, clouds, lidar):
    lc, ls, sharp, flat = clouds[lidar]
    res = _against_checker(oracle, lc, ls, sharp, flat, lidar)
    # the surface scans find both a second and a third point for most queries
    ns = sharp.shape[0]
    assert (res["ind"][ns:, 2] >= 0).mean() > 0.5


@pytest.mark.parametrize("variant", ["rings_permuted", "points_moved", "rings_250_255", "rings_250_255_sorted",
                                     "ring_gaps", "negative_intensity"])
@pytest.mark.parametrize("lidar", list(LIDARS))
def test_reference_search_unordered_rings(oracle, clouds, lidar, variant):
    lc, ls, sharp, flat = clouds[lidar]
    vc, vs = orf.fallback_variants(lc, ls)[variant]
    assert vc.shape == lc.shape and vs.shape == ls.shape
    _against_checker(oracle, vc, vs, sharp, flat, f"{lidar}/{variant}")


def test_reference_scan_edges(oracle):
    """Hand-made clouds (odom_reference.edge_cases): the d^2 = 25 gate of the closest point and of the scans, closest
    points at both ends of the cloud, equidistant candidates on both sides of the closest point, empty query arrays."""
    cases = orf.edge_cases()
    for name, (lc, ls, sharp, flat) in cases.items():
        _against_checker(oracle, lc, ls, sharp, flat, name, dense=False)
    # the cases exercise what they are named after
    s = orf.Search(*cases["gate_closest_at_25"][:2])
    assert s.run(*cases["gate_closest_at_25"][2:])["ind"][0, 0] == -1
    s = orf.Search(*cases["gate_closest_below_25"][:2])
    assert s.run(*cases["gate_closest_below_25"][2:])["ind"][0, 0] == 1
    for name, i1 in (("closest_first", 0), ("closest_last", 49)):
        assert orf.Search(*cases[name][:2]).run(*cases[name][2:])["ind"][0, 0] == i1


def test_ulps_apart():
    a = np.float32(25.0)
    assert orf.ulps_apart(a, np.nextafter(a, np.float32(0))) == 1
    assert orf.ulps_apart(a, a) == 0
    assert math.isfinite(float(orf.ulps_apart(np.float32(1.0), np.float32(2.0))))
