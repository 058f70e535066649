"""GPU parity on randomised configurations (run with -m gpu on an H100): the 240 whole-execute() draws of
tests/cases.py fuzz_config — the four classes x grid / masked / points x every drift kind x anisotropy x exact_values x
moving window, masks and specified-drift arrays also in the transposed orientation the reference tolerates, rasters with
a descending axis, exact hits, 1 x 1 grids, as few as 8 data points — through the C ABI against the outputs of the
unmodified imported reference (tests/golden/ref_fuzz.npz, make_golden.py fuzz). The reference's own kriging matrices of
these draws have 2-norm condition numbers <= 1.3e5 (stored per draw), so the fp64 tolerance of SURVEY.md §8(d) applies
unchanged: rtol = 1e-5, atol = 1e-5 * max|ref| on z and sigma^2. The same draws run through the host wrappers on the CPU
emulator in tests/test_host_execute_emulated.py."""
import os
import warnings

import numpy as np
import pytest

import cases
from conftest import GOLDEN, assert_parity

pytestmark = pytest.mark.gpu
R64 = 1e-5


@pytest.fixture(scope="module")
def pk():
    import pykrige_b200
    return pykrige_b200


@pytest.fixture(scope="module")
def ref_fuzz():
    return np.load(os.path.join(GOLDEN, "ref_fuzz.npz"))


@pytest.mark.parametrize("t", range(cases.N_FUZZ))
def test_randomised_configurations_match_reference(pk, t, ref_fuzz):
    c = cases.fuzz_config(t)
    if c is None or "%d/z" % t not in ref_fuzz.files:
        pytest.skip("over-determined draw")
    assert float(ref_fuzz["%d/cond" % t]) < 1e8
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model = getattr(pk, c["cls"])(*c["data"], **c["kw"])
        z, ss = model.execute(c["style"], *c["pts"], backend="cuda", **c["ekw"])
    zr, sr, mr = ref_fuzz["%d/z" % t], ref_fuzz["%d/ss" % t], ref_fuzz["%d/mask" % t]
    assert z.shape == zr.shape and ss.shape == sr.shape, c["text"]
    if c["style"] == "masked":
        assert np.array_equal(np.ma.getmaskarray(z), mr) and np.array_equal(np.ma.getmaskarray(ss), mr), c["text"]
        keep = ~mr
        z, ss, zr, sr = np.ma.getdata(z)[keep], np.ma.getdata(ss)[keep], zr[keep], sr[keep]
    if zr.size:
        assert_parity(np.ravel(z), np.ravel(zr), R64, "draw %d %s z" % (t, c["text"]))
        assert_parity(np.ravel(ss), np.ravel(sr), R64, "draw %d %s ss" % (t, c["text"]))
    model._kb_handle.close()
