"""Timing of leave_group_out() (DESIGN.md §5f).

    python scripts/lgo_timing.py [--reps 5] [--out results.json]

Config 2 (N = 5000, exponential [1, 300, 0.05]) from the held factorisation, for 5 and 10 random folds and a 10 x 10
block grid: the whole kb200_lgo call (host clock), and from kb200_last_timings the Gram product G = W^T W
(trtri_ms), the group solves (finalize_ms: alpha, the blocks and their inverses) and all of its kernels (solve_ms).
The CPU brute force of one reduced fold (5 folds: a ~4000-station matrix, scipy.linalg.inv, inverse x RHS, as the
reference's GridSearchCV route kriges). Config 5 (N = 1e5, exponential [1, 50, 0.05], k = 64): the moving-window
leave-group-out of every station with a 20 x 20 block grid. Medians of --reps repeats after one warm-up. The card name
and power limit are read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import cases  # noqa: E402
import pykrige_b200 as pk  # noqa: E402
from loo_timing import card, median_s  # noqa: E402
from oracle import krige_oracle as ko  # noqa: E402


def blocks(X, nb):
    lo, hi = X.min(0), X.max(0)
    c = np.minimum((nb * (X - lo) / (hi - lo)).astype(int), nb - 1)
    return c[:, 0] * nb + c[:, 1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rows = {}
    X, val = cases.synth_data(1002, 5000, 2)
    n = X.shape[0]
    model = pk.OrdinaryKriging(X[:, 0], X[:, 1], val, variogram_model="exponential",
                               variogram_parameters=[1.0, 300.0, 0.05])
    h = model._ensure_problem("float64")
    layouts = {"kfold5": np.random.default_rng(5).permutation(np.arange(n) % 5),
               "kfold10": np.random.default_rng(10).permutation(np.arange(n) % 10),
               "blocks10x10": blocks(X, 10)}
    for name, groups in layouts.items():
        dense = np.unique(groups, return_inverse=True)[1].astype(np.int32)
        ng = int(dense.max()) + 1
        h.lgo(dense, ng, n)
        h.reset_counters()
        rows["cfg2_%s_call_s" % name] = median_s(lambda: h.lgo(dense, ng, n), a.reps)
        t = h.timings()
        k = a.reps + 1
        rows["cfg2_%s_gram_ms" % name] = t["trtri_ms"] / k
        rows["cfg2_%s_group_solves_ms" % name] = t["finalize_ms"] / k
        rows["cfg2_%s_kernels_ms" % name] = t["solve_ms"] / k
        rows["cfg2_%s_factorisations" % name] = t["cholesky_ms"]
    keep = layouts["kfold5"] != 0
    m = [0.95, 300.0, 0.05]

    def one_fold():
        A = ko.kriging_matrix(X[keep], "exponential", m)
        ko.exec_vector(A, X[keep], X[~keep], val[keep], "exponential", m)
    rows["cpu_one_reduced_fold_kfold5_s"] = median_s(one_fold, 2)
    X5, v5 = cases.synth_data(1005, 100000, 2)
    m5 = pk.OrdinaryKriging(X5[:, 0], X5[:, 1], v5, variogram_model="exponential", variogram_parameters=[1.0, 50.0, 0.05])
    g5 = blocks(X5, 20)
    rows["cfg5_knn_lgo_k64_blocks20x20_s"] = median_s(lambda: m5.leave_group_out(g5, n_closest_points=64), a.reps)
    rows["cfg5_knn_loo_k64_s"] = median_s(lambda: m5.leave_one_out(n_closest_points=64), a.reps)
    out = dict(card=card(), cfg2=dict(n=5000, model="exponential", params=[1.0, 300.0, 0.05]),
               cfg5=dict(n=100000, k=64, params=[1.0, 50.0, 0.05]), reps=a.reps, rows=rows)
    print(json.dumps(out), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
