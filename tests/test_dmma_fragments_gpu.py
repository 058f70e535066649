"""Per-lane fragment maps of the fp64 mma.sync shapes the solve kernels use (m8n8k4, m16n8k4, m16n8k8, m16n8k16).

One warp loads row-major A, B, C through the maps written in scripts/dmma_rate.cu (the same ones solve.cu and the fp64
packers assume), runs one MMA and stores D through the C map. Small integers keep every product and sum exact, so D must
equal A @ B + C bit for bit; a wrong A, B or C map scrambles it."""
import ctypes
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "scripts", "libdmma_rate.so")
SHAPES = {"m8n8k4": (0, 8, 4), "m16n8k4": (1, 16, 4), "m16n8k8": (2, 16, 8), "m16n8k16": (3, 16, 16)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SHAPES))
def test_fragment_map_exact(name):
    assert os.path.exists(LIB), "scripts/libdmma_rate.so is not built (make -C pykrige_b200/csrc)"
    lib = ctypes.CDLL(LIB)
    lib.dmma_frag_run.argtypes = [ctypes.c_int] + [ctypes.c_void_p] * 4
    shape, m, k = SHAPES[name]
    rng = np.random.default_rng(17 + shape)
    a = rng.integers(-8, 9, size=(m, k)).astype(np.float64)
    b = rng.integers(-8, 9, size=(k, 8)).astype(np.float64)
    c = rng.integers(-64, 65, size=(m, 8)).astype(np.float64)
    d = np.full((m, 8), np.nan)
    err = lib.dmma_frag_run(shape, a.ctypes.data, b.ctypes.data, c.ctypes.data, d.ctypes.data)
    assert err == 0, "cudaError %d" % err
    np.testing.assert_array_equal(d, a @ b + c)
