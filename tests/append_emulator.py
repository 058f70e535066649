"""CPU emulation of kb200_append_data (include/krige_b200.h) — TEST INFRASTRUCTURE ONLY.

`AppendEmulatedHandle` is tests/cv_emulator.py's `CvEmulatedHandle` plus the append entry point with the semantics the
header states: the held global problem grows by m stations, adjusted with the HELD centre and anisotropy (not the
object's new ones), with their values and host drift columns appended; the kriging matrix is rebuilt by the oracle (the
block-row algebra itself is tests/test_append_algebra.py, the kernels tests/test_append_gpu.py). Refusals: no global
problem factored on this handle, the pseudo-inverse, value fields (NotImplementedError); a singular extended matrix
drops the problem and raises numpy.linalg.LinAlgError. Used by tests/test_append_host.py."""
import warnings

import numpy as np
import scipy.linalg

from oracle import krige_oracle as ko
from cv_emulator import CvEmulatedHandle


class AppendEmulatedHandle(CvEmulatedHandle):
    def append_data(self, x, y, z, values, drift_cols=None):
        self.calls.append("append_data")
        p = self.problem
        if p is None or p["knn"] or not getattr(self, "ready", False) or self.from_blob:
            raise NotImplementedError("append: no global problem was factored on this handle")
        if p["pinv"] or self.fields is not None:
            raise NotImplementedError("append: pseudo-inverse / value fields have no append form")
        cols = [np.asarray(x, float), np.asarray(y, float)] + ([np.asarray(z, float)] if p["dim"] == 3 else [])
        m = cols[0].size
        assert m >= 1 and all(c.size == m for c in cols) and np.size(values) == m
        hd = [] if drift_cols is None else [np.asarray(c, float).ravel() for c in drift_cols]
        assert len(hd) == len(p["hd"]) and all(c.size == m for c in hd), "drift_cols is column-major m x n_hd"
        p["X"] = np.vstack([p["X"], np.column_stack(cols)])
        p["values"] = np.concatenate([p["values"], np.asarray(values, float)])
        p["hd"] = [np.concatenate([a, b]) for a, b in zip(p["hd"], hd)]
        if p["geo"]:
            return
        P = self._adjust(p["X"])                      # the held frame
        dcols = [P[:, c] for c in range(p["dim"])] if p["n_rl"] else []
        p["P"] = P
        p["a"] = ko.kriging_matrix(P, p["fn"], p["m"], dcols + p["hd"])
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                scipy.linalg.inv(p["a"])
        except np.linalg.LinAlgError:
            self.problem = None
            self.ready = False
            raise
