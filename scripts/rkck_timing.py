"""Timing of ClassificationKriging.predict with C = 9 classes: the residuals kriged class by class (C - 1 = 8 problems)
against one problem with 8 value fields (execute(values=R), the route krige_residual takes with fixed variogram
parameters).

    python scripts/rkck_timing.py [--reps 3] [--points 1000000] [--out results.json]

Two set-ups, both with a LogisticRegression classifier on four covariates and exponential [1, 300, 0.05]:
  cfg2: N = 5000 stations (the size of config 2), global path (n_closest_points=None);
  cfg5: N = 100000 stations, moving window with k = 64 (config 5's window).
Each is kriged at --points scattered prediction points. Two models are fitted on the same data, one held to the
per-class route; predict() alternates between them. 'first' is the first predict of a model (it includes the
factorisations); the median of --reps further predicts is the steady state, with every factorisation held. The host
clock brackets each call, which ends in a copy of the results to the host. krige_residual of both routes is compared
bit for bit in the same run, and the card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pykrige_b200 as pk  # noqa: E402
from pykrige_b200.ck import ClassificationKriging  # noqa: E402

PARAMS = [1.0, 300.0, 0.05]
N_CLASSES = 9


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def data(n, m, seed):
    rng = np.random.default_rng(seed)
    x = rng.uniform(0.0, 1000.0, size=(n + m, 2))
    p = np.column_stack([x / 1000.0 + rng.normal(scale=0.2, size=(n + m, 2)), rng.normal(size=(n + m, 2))])
    score = 3.0 * p[:, 0] + 2.0 * p[:, 1] + np.sin(x[:, 0] / 150.0) + 0.5 * rng.normal(size=n + m)
    y = np.digitize(score, np.quantile(score[:n], np.linspace(0.0, 1.0, N_CLASSES + 1)[1:-1]))
    return p[:n], x[:n], y[:n].astype(np.float64).reshape(-1, 1), p[n:], x[n:]


def run(label, n, k, m, reps, seed):
    from sklearn.linear_model import LogisticRegression
    p, x, y, pq, xq = data(n, m, seed)
    models = {}
    for route in ("per_class", "shared"):
        ck = ClassificationKriging(classification_model=LogisticRegression(max_iter=500), n_closest_points=k,
                                   variogram_model="exponential", variogram_parameters=PARAMS)
        ck.fit(p, x, y)
        if route == "per_class":
            ck._shares_one_problem = lambda kwargs: False
        models[route] = ck
    assert len(models["shared"].classes_) == N_CLASSES and models["shared"]._shares_one_problem({})
    warm = pk.OrdinaryKriging(x[:, 0], x[:, 1], models["shared"]._residuals[:, 0], variogram_model="exponential",
                              variogram_parameters=PARAMS)
    warm.execute("points", xq[:1000, 0], xq[:1000, 1], n_closest_points=k)      # module load, outside the timings

    def timed(route):
        t0 = time.perf_counter()
        pred = models[route].predict(pq, xq)
        return time.perf_counter() - t0, pred

    first, preds, times = {}, {}, {"per_class": [], "shared": []}
    for route in ("per_class", "shared"):
        first[route], preds[route] = timed(route)
    for _ in range(reps):
        for route in ("per_class", "shared"):
            times[route].append(timed(route)[0])
    t0 = time.perf_counter()
    rs = models["shared"].krige_residual(xq)
    resid_shared_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    rp = models["per_class"].krige_residual(xq)
    resid_per_class_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    models["shared"].classification_model.predict_proba(pq)
    proba_s = time.perf_counter() - t0
    row = dict(setup=label, n_stations=n, n_closest_points=k, points=m, classes=N_CLASSES,
               first_predict_s={r: round(first[r], 4) for r in first},
               predict_s={r: round(float(np.median(times[r])), 4) for r in times},
               predict_s_all={r: [round(t, 4) for t in times[r]] for r in times},
               krige_residual_s=dict(per_class=round(resid_per_class_s, 4), shared=round(resid_shared_s, 4)),
               classifier_predict_proba_s=round(proba_s, 4),
               residuals_bit_identical=bool(np.array_equal(rs, rp)),
               predictions_identical=bool(np.array_equal(preds["shared"], preds["per_class"])))
    row["predict_speedup"] = round(row["predict_s"]["per_class"] / row["predict_s"]["shared"], 3)
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--points", type=int, default=1000000)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    a = ap.parse_args()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        rows = [run("cfg2_global", 5000, None, a.points, a.reps, 2),
                run("cfg5_moving_window_k64", 100000, 64, a.points, a.reps, 5)]
    out = dict(card=card(), model="exponential", params=PARAMS, reps=a.reps, rows=rows)
    print(json.dumps({"card": out["card"]}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
