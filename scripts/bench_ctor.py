"""Timings of the constructor-side device kernels and of pseudo_inv=True (SURVEY.md §8f next-2 / next-4) on
one H100, next to the host (numpy/scipy) route of the same repo on the box's CPU. One JSON line per item.

    python scripts/bench_ctor.py [ev,stats,pinv] [small]
"""
import json
import os
import sys
import time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases  # noqa: E402
import pykrige_b200 as pk  # noqa: E402
from pykrige_b200 import core, _cabi  # noqa: E402


def wall(fn, reps=1):
    best = 1e30
    out = None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        best = min(best, time.perf_counter() - t0)
    return best, out


def main():
    items = set((sys.argv[1] if len(sys.argv) > 1 else "ev,stats,pinv").split(","))
    small = len(sys.argv) > 2 and sys.argv[2] == "small"          # short run for an ncu launch list
    h = _cabi.aux_handle()
    rng = np.random.default_rng(1)
    # ---- experimental variogram ------------------------------------------------------------------
    for n, host in (((20000, False),) if small else ((5000, True), (20000, True), (100000, False))):
        if "ev" not in items:
            break
        X = rng.uniform(0.0, 1000.0, (n, 2))
        y = rng.normal(0.0, 1.0, n) + 0.01 * X[:, 0]
        h.experimental_variogram(X[:512], y[:512], 6)                     # warm-up
        t_dev, (cnt, sd, sg, dmin, dmax) = wall(lambda: h.experimental_variogram(X, y, 6), reps=3)
        rec = {"item": "experimental_variogram", "n": n, "pairs": n * (n - 1) // 2, "nlags": 6,
               "device_s": t_dev, "pairs_per_s": n * (n - 1) / 2 / t_dev}
        if host:
            t_host, (lags_h, semi_h) = wall(lambda: core._experimental_variogram(X, y, 6, device=False))
            keep = cnt > 0
            rec.update(host_s=t_host, speedup=t_host / t_dev,
                       max_rel_lag=float(np.max(np.abs(sd[keep] / cnt[keep] / lags_h - 1.0))),
                       max_rel_semi=float(np.max(np.abs(sg[keep] / cnt[keep] / semi_h - 1.0))))
        print(json.dumps(rec), flush=True)
    # ---- cross-validation statistics ---------------------------------------------------------------
    for n, host_n in (((5000, 0),) if small else ((5000, 400), (20000, 0))):
        if "stats" not in items:
            break
        xyz, val = cases.synth_data(808, n, 2)
        ok = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="exponential",
                                variogram_parameters=[1.0, 300.0, 0.05])
        hh = ok._ensure_problem("float64")
        t_stat, (delta, sigma) = wall(lambda: hh.statistics(n), reps=3)
        ok._kb_key = None
        t_all, _ = wall(lambda: (ok._ensure_problem("float64"), hh.statistics(n)))
        rec = {"item": "statistics", "n": n, "device_stats_only_s": t_stat, "device_factor_plus_stats_s": t_all}
        if host_n:
            t_host, (d, s, e) = wall(lambda: core._find_statistics(xyz[:host_n], val[:host_n],
                                                                   ok.variogram_function, ok.variogram_model_parameters))
            # the reference's loop costs sum_i i^3 ~ n^4/4: extrapolate from host_n to n
            rec.update(host_n=host_n, host_s_at_host_n=t_host, host_s_extrapolated=t_host * (n / host_n) ** 4,
                       max_abs_delta_diff=float(np.max(np.abs(delta[1:host_n] - d))))
        print(json.dumps(rec), flush=True)
    # ---- pseudo_inv=True -----------------------------------------------------------------------------
    import scipy.linalg
    from scipy.spatial.distance import cdist
    for n in ((300,) if small else (500, 1000, 2000, 4000)):
        if "pinv" not in items:
            break
        xyz, val = cases.synth_data(4242, n, 2)
        for q in range(10):
            xyz[n - 1 - q] = xyz[2 * q]
        params = [1.0, 250.0, 0.0]
        pts = cases.synth_points(4242, 2000, 2, xyz)
        m = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="exponential", variogram_parameters=params,
                               pseudo_inv=True)
        t_dev, (z, ss) = wall(lambda: m.execute("points", pts[:, 0], pts[:, 1], backend="cuda"))
        tm = m._cuda_handle().timings()
        rec = {"item": "pseudo_inv", "n": n, "device_total_s": t_dev, "launches": tm["launches"],
               "z_mean": float(np.mean(z)), "ss_mean": float(np.mean(ss))}
        if n <= 2000:
            # what the reference spends on the same step: scipy.linalg.pinv of the (n+1)^2 kriging matrix
            a = np.zeros((n + 1, n + 1))
            a[:n, :n] = -m.variogram_function(m.variogram_model_parameters, cdist(xyz, xyz))
            np.fill_diagonal(a, 0.0)
            a[n, :n] = 1.0
            a[:n, n] = 1.0
            t_host, _ = wall(lambda: scipy.linalg.pinv(a))
            rec.update(host_scipy_pinv_s=t_host)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
