"""CPU tests of the extended-precision reference (oracle.krige_oracle.exec_vector_refined) that the GPU boundary sweep
(test_solve_boundaries_gpu.py) judges the solve kernels by: on small systems it must equal a 40-digit mpmath solve of
the same fp64 matrix and RHS to fp64 rounding, and the reference's own fp64 inverse (exec_vector) must agree with it
to kappa * eps."""
import mpmath
import numpy as np
import pytest
from scipy.spatial.distance import cdist

import cases
from conftest import assert_parity
from oracle import krige_oracle as ko

EPS64 = np.finfo(np.float64).eps

# (name, n, model, full-form params, regional_linear, functional drift, anisotropy (scaling, angle), exact_values)
SYSTEMS = [
    ("ok_exponential", 20, "exponential", [1.0, 300.0, 0.05], False, 0, None, True),
    ("ok_linear_nonexact", 33, "linear", [0.004, 0.05], False, 0, None, False),
    ("uk_rl_spherical_aniso", 30, "spherical", [1.0, 400.0, 0.05], True, 0, (1.7, 30.0), True),
    ("uk_rl_func_exponential", 40, "exponential", [1.0, 250.0, 0.02], True, 3, None, True),
]
_FUNCS = [lambda u, v: u * v, lambda u, v: u * u - v * v, lambda u, v: np.cos(2.0 * u)]


def _system(name, n, model, params, rl, nfunc, aniso, exact):
    seed = 900 + n
    xyz, val = cases.synth_data(seed, n, 2)
    pts = cases.synth_points(seed, 12, 2, xyz, n_hits=2)          # 12 scattered points, 2 exact hits
    center = (xyz.max(axis=0) + xyz.min(axis=0)) / 2.0
    scaling, angle = ([aniso[0]], [aniso[1]]) if aniso else ([1.0], [0.0])
    P = ko.adjust_for_anisotropy(xyz, center, scaling, angle)
    Q = ko.adjust_for_anisotropy(pts, center, scaling, angle)
    dd, pd = ([P[:, 0], P[:, 1]], [Q[:, 0], Q[:, 1]]) if rl else ([], [])
    for f in _FUNCS[:nfunc]:
        dd.append(f((P[:, 0] - 500.0) / 500.0, (P[:, 1] - 500.0) / 500.0))
        pd.append(f((Q[:, 0] - 500.0) / 500.0, (Q[:, 1] - 500.0) / 500.0))
    m = ko.stored_parameters(model, params)
    return ko.kriging_matrix(P, model, m, dd), P, Q, val, m, pd


def _mpmath_solve(a, P, Q, values, model, m, exact, drift_pts):
    """The same system at 40 significant digits: every fp64 entry converts exactly, the LU runs in mpmath."""
    n = P.shape[0]
    bd = cdist(Q, P)
    b = np.zeros((Q.shape[0], a.shape[0]))
    b[:, :n] = -ko.variogram(model, m, bd)
    if exact:
        b[:, :n][bd <= ko.EPS] = 0.0
    for i, col in enumerate(drift_pts):
        b[:, n + i] = col
    b[:, -1] = 1.0
    with mpmath.workdps(40):
        A = mpmath.matrix(a.tolist())
        z, ss = [], []
        for j in range(b.shape[0]):
            bj = mpmath.matrix(b[j].tolist())
            x = mpmath.lu_solve(A, bj)
            z.append(float(mpmath.fsum(x[i] * mpmath.mpf(values[i]) for i in range(n))))
            ss.append(float(-mpmath.fsum(x[i] * bj[i] for i in range(a.shape[0]))))
    return np.array(z), np.array(ss)


@pytest.mark.parametrize("sysdef", SYSTEMS, ids=[s[0] for s in SYSTEMS])
def test_refined_reference_matches_mpmath(sysdef):
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("np.longdouble has no extended mantissa on this platform")
    exact = sysdef[7]
    a, P, Q, val, m, pd = _system(*sysdef)
    z, ss, kappa = ko.exec_vector_refined(a, P, Q, val, sysdef[2], m, exact, pd)
    zm, sm = _mpmath_solve(a, P, Q, val, sysdef[2], m, exact, pd)
    assert_parity(z, zm, 1e-15, sysdef[0] + " refined z vs mpmath")
    assert_parity(ss, sm, 1e-15, sysdef[0] + " refined ss vs mpmath")
    if exact:                                       # the exact hits: z = the datum, sigma^2 = 0
        np.testing.assert_allclose(z[-2:], val[:2], rtol=1e-15)
        assert np.max(np.abs(ss[-2:])) <= 1e-15 * np.max(np.abs(ss))
    # the reference's fp64 inverse x RHS carries kappa * eps relative to the exact solution, no more
    ze, se = ko.exec_vector(a, P, Q, val, sysdef[2], m, exact, pd)
    assert_parity(ze, z, kappa * EPS64, sysdef[0] + " exec_vector z vs refined (kappa %.2e)" % kappa)
    assert_parity(se, ss, kappa * EPS64, sysdef[0] + " exec_vector ss vs refined (kappa %.2e)" % kappa)


def test_refined_reference_refines():
    """On an ill-conditioned system (gaussian model, zero nugget, two pairs of points about a metre apart in a 1 km
    box) the plain fp64 solve is off by ~kappa * eps, while the refined one stays within kappa * eps(longdouble) of
    mpmath: the refinement steps do the work, not the fp64 LU."""
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("np.longdouble has no extended mantissa on this platform")
    xyz, val = cases.synth_data(41, 30, 2)
    xyz[1] = xyz[0] + [0.5, 0.5]
    xyz[3] = xyz[2] + [0.0, 1.0]
    pts = cases.synth_points(41, 8, 2, xyz, n_hits=1)
    m = ko.stored_parameters("gaussian", [1.0, 400.0, 0.0])
    a = ko.kriging_matrix(xyz, "gaussian", m)
    z, ss, kappa = ko.exec_vector_refined(a, xyz, pts, val, "gaussian", m)
    z0, s0, _ = ko.exec_vector_refined(a, xyz, pts, val, "gaussian", m, steps=0)
    zm, sm = _mpmath_solve(a, xyz, pts, val, "gaussian", m, True, ())
    assert kappa > 1e6
    R = kappa * float(np.finfo(np.longdouble).eps)
    assert_parity(z, zm, R, "ill-conditioned refined z vs mpmath")
    assert_parity(ss, sm, R, "ill-conditioned refined ss vs mpmath")
    assert np.max(np.abs(z0 - zm)) > 1e3 * np.max(np.abs(z - zm))
