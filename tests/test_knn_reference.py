"""CPU tests of the moving-window reference (tests/knn_reference.py) that the GPU sweep test_knn_boundaries_gpu.py judges
the kernel by: its neighbour sets are cKDTree's where there are no ties and follow (d^2, index) where there are, its
ambiguity flag fires on a near-tie, its outputs equal the oracle's moving window (oracle.krige_oracle.
exec_moving_window) to kappa * eps, its weights equal a 40-digit mpmath solve of the same system, and its mirror of the
kernel's shared-memory footprint gives the k limit and the points per CTA of csrc/knn.cu."""
import mpmath
import numpy as np
import pytest
from scipy.spatial import cKDTree

import cases
import knn_reference as kr
from conftest import assert_parity
from oracle import krige_oracle as ko
from pykrige_b200.core import anisotropy_matrix

EPS64 = np.finfo(np.float64).eps


def test_no_ties_sets_and_outputs_match_the_oracle():
    xyz, val = cases.synth_data(71, 400, 2)
    pts = cases.synth_points(71, 30, 2, xyz, n_hits=4)
    m = ko.stored_parameters("exponential", [1.0, 300.0, 0.05])
    for k in (2, 9, 64, 156):
        _, idx = cKDTree(xyz).query(pts, k=k)
        idx = idx.reshape(pts.shape[0], -1)
        for i in range(pts.shape[0]):
            nb = kr.neighbours(xyz, pts[i], k)
            assert not nb.flagged
            assert np.array_equal(nb.sel, np.sort(idx[i]))
        z, ss, kappa, flagged = kr.moving_window(xyz, pts, val, "exponential", m, k)
        zo, so = ko.exec_moving_window(xyz, pts, val, "exponential", m, k)
        R = 8.0 * float(np.max(kappa)) * EPS64
        assert not flagged.any()
        assert_parity(z, zo, R, "k=%d z" % k)
        assert_parity(ss, so, R, "k=%d ss" % k)


def test_geographic_matches_the_oracle():
    rng = np.random.default_rng(5)
    P = np.column_stack([rng.uniform(-180.0, 180.0, 300), np.degrees(np.arcsin(rng.uniform(-1.0, 1.0, 300)))])
    val = rng.normal(size=300)
    Q = np.array([[179.99, 10.0], [-179.99, -10.0], [0.0, 89.9], [33.0, -89.9], [12.0, 3.0]])
    m = ko.stored_parameters("exponential", [1.0, 40.0, 0.02])
    z, ss, kappa, flagged = kr.moving_window(P, Q, val, "exponential", m, 12, geo=True)
    zo, so = ko.krige_geographic(P, val, "exponential", m, Q, n_closest_points=12)
    assert not flagged.any()
    R = 8.0 * float(np.max(kappa)) * EPS64
    assert_parity(z, zo, R, "geo z")
    assert_parity(ss, so, R, "geo ss")


def test_lattice_ties_follow_distance_then_index():
    g = np.arange(9.0)
    P = np.column_stack([np.tile(g, 9), np.repeat(g, 9)])          # index = 9 y + x
    q = np.array([4.0, 4.0])
    nb = kr.neighbours(P, q, 3)                                    # the node and two of its four unit neighbours
    assert not nb.flagged
    assert np.array_equal(nb.sel, [4 + 9 * 3, 3 + 9 * 4, 4 + 9 * 4])
    assert np.array_equal(nb.band, np.sort([4 + 9 * 3, 3 + 9 * 4, 5 + 9 * 4, 4 + 9 * 5])) and nb.need == 2
    nb = kr.neighbours(P, np.array([4.5, 4.5]), 2)                 # cell centre: four at the same distance
    assert np.array_equal(nb.sel, [4 + 9 * 4, 5 + 9 * 4])
    nb = kr.neighbours(P, q, 3, exclude=[3 + 9 * 4, 4 + 9 * 4])    # leave-group-out of two of them
    assert np.array_equal(nb.sel, [4 + 9 * 3, 5 + 9 * 4, 4 + 9 * 5])
    assert nb.accepts([4 + 9 * 5, 4 + 9 * 3, 5 + 9 * 4]) and not nb.accepts([4 + 9 * 3, 5 + 9 * 4, 3 + 9 * 4])


def test_ambiguity_flag_fires_on_a_near_tie():
    P = np.array([[0.0, 0.0], [1.0, 0.0], [0.0, 1.0 + 1e-14], [3.0, 3.0]])
    nb = kr.neighbours(P, np.zeros(2), 2)
    assert nb.flagged and np.array_equal(nb.must, [0]) and np.array_equal(nb.band, [1, 2]) and nb.need == 1
    assert nb.accepts([0, 1]) and nb.accepts([2, 0]) and not nb.accepts([1, 2])
    P[2, 1] = 1.0 + 1e-9                                           # far outside rounding: decided
    nb = kr.neighbours(P, np.zeros(2), 2)
    assert not nb.flagged and np.array_equal(nb.sel, [0, 1])
    P[2, 1] = 1.0                                                  # an exact tie: decided by index
    nb = kr.neighbours(P, np.zeros(2), 2)
    assert not nb.flagged and np.array_equal(nb.sel, [0, 1])


def test_device_frame_is_the_oracle_map():
    rng = np.random.default_rng(3)
    for dim, scaling, angle, off in ((2, [5.0], [35.0], (5e5, 5e6)), (3, [2.0, 0.5], [20.0, 35.0, 50.0], (0, 0, 0))):
        X = rng.uniform(0.0, 30.0, (200, dim)) + np.asarray(off)
        c = (X.max(axis=0) + X.min(axis=0)) / 2.0
        A = kr.device_frame(X, c, anisotropy_matrix(dim, scaling, angle))
        B = ko.adjust_for_anisotropy(X, c, scaling, angle)
        assert np.max(np.abs(A - B)) <= 8.0 * EPS64 * np.max(np.abs(B))


def _mpmath_weights(a, b):
    with mpmath.workdps(40):
        x = mpmath.lu_solve(mpmath.matrix(a.tolist()), mpmath.matrix(b.tolist()))
        return np.array([float(x[i]) for i in range(a.shape[0])])


@pytest.mark.parametrize("model,params,k,close", [("exponential", [1.0, 300.0, 0.05], 12, False),
                                                  ("spherical", [1.0, 200.0, 0.0], 20, False),
                                                  ("linear", [0.004, 0.05], 16, False),
                                                  ("gaussian", [1.0, 400.0, 0.0], 16, True)])
def test_refined_weights_match_mpmath(model, params, k, close):
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("np.longdouble has no extended mantissa on this platform")
    xyz, val = cases.synth_data(90 + k, 60, 2)
    if close:                                                      # two pairs 0.1 apart in 1 km: kappa ~ 1e10
        xyz[1] = xyz[0] + [0.07, 0.07]
        xyz[3] = xyz[2] + [0.0, 0.1]
    q = xyz[0] + np.array([3.0, -2.0])
    m = ko.stored_parameters(model, params)
    nb = kr.neighbours(xyz, q, k)
    lam, z, ss, kappa = kr.local_solution(xyz[nb.sel], q, val[nb.sel], model, m, True)
    a, b = kr.local_system(xyz[nb.sel], q, model, m, True, False)
    x = _mpmath_weights(a, b)
    if close:
        assert kappa > 1e9
    R = max(kappa * float(np.finfo(np.longdouble).eps), 2.0 * EPS64)
    assert np.max(np.abs(lam - x[:k])) <= R * np.max(np.abs(x[:k]))
    with mpmath.workdps(40):
        zm = float(mpmath.fsum(mpmath.mpf(x[i]) * mpmath.mpf(val[nb.sel][i]) for i in range(k)))
    assert abs(z - zm) <= R * abs(zm) * 10.0
    assert abs(ss - float(-x @ b)) <= R * 10.0 * abs(ss) + 1e-15


def test_shared_memory_mirror():
    # by hand from knn.cu: k = 64 tiled Cholesky in 2-D, one field: 8 x 9 / 2 + 8 + 1 tiles of 64 doubles, four
    # per-neighbour arrays of 64, two spare doubles -> 25104 bytes, 9 points per CTA;
    # k = 156 LU: 156 x 157 + 7 x 156 + 2 doubles -> 204688 bytes, one point per CTA
    assert kr.smem_per_warp(64, 1, 0, 1) == 25104 and kr.points_per_cta(64, 1, 0, 1) == 9
    assert kr.smem_per_warp(156, 0, 0, 1) == 204688 and kr.points_per_cta(156, 0, 0, 1) == 1
    assert kr.points_per_cta(8, 1, 0, 1) == 10
    assert kr.k_supported(156) and not kr.k_supported(157)
    assert max(k for k in range(2, 400) if kr.k_supported(k)) == 156
