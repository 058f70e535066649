"""Timing of leave_one_out() (DESIGN.md §5e).

    python scripts/loo_timing.py [--reps 5] [--out results.json]

Config 2 (N = 5000, exponential [1, 300, 0.05]): the factorisation (kb200_set_problem, host clock around a call that ends
in a device synchronise), the leave-one-out of every station from the held factorisation at V = 1 and V = 64 value
fields (host clock around kb200_loo, and the device time of its kernels from kb200_last_timings), and the whole
leave_one_out() call of a fresh object, which includes its factorisation. Config 5 (N = 1e5, exponential [1, 50, 0.05],
k = 64): the moving-window leave-one-out of every station. The CPU brute force: one reduced solve the way the reference
kriges (the N - 1 station matrix, scipy.linalg.inv, inverse x RHS), multiplied by N and labelled as extrapolated.
Medians of --reps repeats after one warm-up. The card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases  # noqa: E402
import pykrige_b200 as pk  # noqa: E402
from oracle import krige_oracle as ko  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def median_s(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), [round(t, 5) for t in ts]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rows = {}
    X, val = cases.synth_data(1002, 5000, 2)
    kw = dict(variogram_model="exponential", variogram_parameters=[1.0, 300.0, 0.05])
    n = X.shape[0]
    model = pk.OrdinaryKriging(X[:, 0], X[:, 1], val, **kw)
    F = 50.0 + 10.0 * np.random.default_rng(0).standard_normal((n, 64))

    def factor():
        model._kb_key = None                       # force kb200_set_problem
        model._ensure_problem("float64")
    rows["cfg2_factorisation_s"] = median_s(factor, a.reps)
    for V in (1, 64):
        h = model._ensure_problem("float64", fields=None if V == 1 else np.ascontiguousarray(F.T))
        h.loo(n)
        h.reset_counters()
        rows["cfg2_loo_V%d_s" % V] = median_s(lambda: h.loo(n), a.reps)
        rows["cfg2_loo_V%d_kernels_ms" % V] = h.timings()["solve_ms"] / (a.reps + 1)
    rows["cfg2_leave_one_out_call_s"] = median_s(
        lambda: pk.OrdinaryKriging(X[:, 0], X[:, 1], val, **kw).leave_one_out(), a.reps)
    # CPU brute force: one reduced problem as the reference kriges it, x N (extrapolated, not measured for N folds)
    P = X
    keep = np.arange(n) != 0
    m = [0.95, 300.0, 0.05]

    def one_fold():
        A = ko.kriging_matrix(P[keep], "exponential", m)
        ko.exec_vector(A, P[keep], P[:1], val[keep], "exponential", m)
    t1, all1 = median_s(one_fold, 2)
    rows["cpu_one_reduced_solve_s"] = (t1, all1)
    rows["cpu_brute_force_extrapolated_s"] = t1 * n
    # config 5: moving window, every station
    X5, v5 = cases.synth_data(1005, 100000, 2)
    m5 = pk.OrdinaryKriging(X5[:, 0], X5[:, 1], v5, variogram_model="exponential", variogram_parameters=[1.0, 50.0, 0.05])
    rows["cfg5_knn_loo_k64_s"] = median_s(lambda: m5.leave_one_out(n_closest_points=64), a.reps)
    out = dict(card=card(), cfg2=dict(n=5000, model="exponential", params=[1.0, 300.0, 0.05]),
               cfg5=dict(n=100000, k=64, params=[1.0, 50.0, 0.05]), reps=a.reps, rows=rows,
               w_bytes_cfg2=5000 * 5000 / 2 * 8)
    print(json.dumps(out), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
