"""Timing of execute(values=...) on config 2 (N = 5000, exponential [1, 300, 0.05], 1000 x 1000 grid).

    python scripts/fields_timing.py [--reps 3] [--out results.json]

For V in (1, 8, 32, 64) value fields in ONE call, and for V = 8 as eight single-field calls (eight objects, what a user
had to do before): the solve-kernel time (kb200_last_timings[4], summed over the call's launches), the whole-call time
(host clock around execute(), which ends in a device synchronise; it includes the factorisation, since every repeat
passes new values) and field-points/s = V * 1e6 / whole-call time. Medians of --reps repeats after one warm-up call
per variant. The card name and power limit are read in the same run."""
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

PARAMS = [1.0, 300.0, 0.05]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    a = ap.parse_args()
    xyz, val = cases.synth_data(1002, 5000, 2)
    g = np.linspace(0.0, 1000.0, 1000)
    npts = g.size * g.size
    rng = np.random.default_rng(0)
    base = 50.0 + 10.0 * rng.standard_normal((5000, 64))

    def make(z):
        return pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], z, variogram_model="exponential", variogram_parameters=PARAMS)

    model = make(val)
    rows = []

    def timed(fn):
        t0 = time.perf_counter()
        solve = fn()
        return time.perf_counter() - t0, solve

    def one_call(V, rep):
        F = base[:, :V] + rep                           # new values every repeat: a new problem, factorised again
        model._cuda_handle().reset_counters()
        z, ss = model.execute("grid", g, g, values=F)
        assert z.shape == (V, 1000, 1000)
        return model._cuda_handle().timings()["solve_ms"]

    def singles(V, rep):
        solve = 0.0
        for v in range(V):
            m = make(base[:, v] + rep)
            z, ss = m.execute("grid", g, g)
            solve += m._cuda_handle().timings()["solve_ms"]
        return solve

    for label, V, fn in [("fields", 1, one_call), ("fields", 8, one_call), ("fields", 32, one_call),
                         ("fields", 64, one_call), ("single_calls", 8, singles)]:
        timed(lambda: fn(V, -1.0))                      # warm-up
        res = [timed(lambda r=r: fn(V, float(r))) for r in range(a.reps)]
        wall = float(np.median([r[0] for r in res]))
        solve = float(np.median([r[1] for r in res]))
        row = dict(kind=label, V=V, call_s=round(wall, 4), solve_ms=round(solve, 2),
                   field_points_per_s=round(V * npts / wall, 1), call_s_all=[round(r[0], 4) for r in res])
        rows.append(row)
        print(json.dumps(row), flush=True)
    out = dict(card=card(), n=5000, grid="1000x1000", model="exponential", params=PARAMS, reps=a.reps, rows=rows)
    v1 = next(r for r in rows if r["kind"] == "fields" and r["V"] == 1)
    v32 = next(r for r in rows if r["kind"] == "fields" and r["V"] == 32)
    out["v32_over_v1_call"] = round(v32["call_s"] / v1["call_s"], 3)
    out["v32_over_v1_solve"] = round(v32["solve_ms"] / v1["solve_ms"], 3)
    print(json.dumps({k: out[k] for k in ("card", "v32_over_v1_call", "v32_over_v1_solve")}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
