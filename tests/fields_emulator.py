"""CPU emulation of kb200_set_values (include/krige_b200.h) — TEST INFRASTRUCTURE ONLY.

`FieldsEmulatedHandle` is tests/abi_emulator.py's `EmulatedHandle` plus the value-fields entry point: the next problem
kriges the V given value vectors instead of its own, each with the oracle exactly like a single-field problem, and
the execute methods return z as V consecutive blocks of the point count and sigma^2 once. The refusals of the header
(dtype other than float64, pseudo-inverse, factor blob, n mismatch) are restated. Used by tests/test_fields_host.py."""
import numpy as np

from abi_emulator import EmulatedHandle


class FieldsEmulatedHandle(EmulatedHandle):
    fields = None
    n_fields = 0

    def set_values(self, fields):
        """kb200_set_values: fields = (V, n) or None; resets the problem state."""
        from pykrige_b200 import _cabi
        self.calls.append("set_values")
        self.problem = None
        if fields is None:
            self.fields, self.n_fields = None, 0
            return
        f = np.asarray(fields, dtype=np.float64)
        if f.ndim != 2 or not 1 <= f.shape[0] <= _cabi.MAX_FIELDS or f.shape[1] < 1 or not np.all(np.isfinite(f)):
            raise ValueError("kb200_set_values: 1 <= n_fields <= KB200_MAX_FIELDS, n >= 1, finite values")
        self.fields, self.n_fields = f.copy(), f.shape[0]

    def _describe(self, knn, dim, x, y, z, values, center, aniso, model, vparams, exact_values, eps, n_rl, drift_data):
        if self.fields is not None and self.fields.shape[1] != np.size(x):
            raise ValueError("kb200_set_values: the fields and the problem differ in n")
        super()._describe(knn, dim, x, y, z, values, center, aniso, model, vparams, exact_values, eps, n_rl,
                          drift_data)

    def set_problem(self, dim, dtype, x, y, z, values, center, aniso, model, vparams, exact_values, eps,
                    n_rl=0, drift_data=None):
        if self.fields is not None and (dtype != 0 or self.pinv):
            raise NotImplementedError("value fields run in float64 only, not with pseudo_inv=True")
        super().set_problem(dim, dtype, x, y, z, values, center, aniso, model, vparams, exact_values, eps,
                            n_rl=n_rl, drift_data=drift_data)

    def describe_problem(self, *args, **kwargs):
        if self.fields is not None:
            raise NotImplementedError("value fields have no factor-blob form")
        return super().describe_problem(*args, **kwargs)

    def _per_field(self, run):
        """run() -> (z, ss) with the problem's values; with fields once per field, z concatenated, ss of the first."""
        if self.fields is None:
            return run()
        own = self.problem["values"]
        out = []
        try:
            for f in self.fields:
                self.problem["values"] = f
                out.append(run())
        finally:
            self.problem["values"] = own
        return np.concatenate([o[0] for o in out]), out[0][1]

    def _krige(self, Q_orig, drift_pts):
        return self._per_field(lambda: EmulatedHandle._krige(self, Q_orig, drift_pts))

    def _knn(self, k, Q_orig):
        return self._per_field(lambda: EmulatedHandle._knn(self, k, Q_orig))
