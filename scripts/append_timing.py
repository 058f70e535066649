"""add_data() + the first execute() against a new object's construction + first execute(), on one GPU (DESIGN.md §5g).

For each N and m: an OrdinaryKriging object on N stations (exponential variogram, fixed parameters) has executed once,
so the device holds its factorisation; the timed call is add_data(m stations) followed by execute() of 1024 points.
The comparison builds a new object on the N + m stations and runs the same execute(), which assembles and factors
everything again. Host wall clock around calls that end in a device synchronise (execute() returns host arrays);
the two arms alternate, each repeated --reps times, and the median is reported together with the relative difference
of their results. The GPU's name, power limit and SM clock limit are read in the same run.

    python scripts/append_timing.py [--sizes 5000 20000 30000] [--m 1 16 64 256] [--reps 3] [--out results.json]
"""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PARAMS = {"psill": 1.0, "range": 300.0, "nugget": 0.05}


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                                        "--format=csv,noheader"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return "unknown (%s)" % e


def data(N, m, seed=0):
    rng = np.random.default_rng(seed)
    xy = rng.uniform(0.0, 1000.0, size=(N + m, 2))
    val = np.sin(xy[:, 0] / 150.0) * np.cos(xy[:, 1] / 200.0) + rng.normal(0.0, 0.1, N + m)
    return xy, val


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[5000, 20000, 30000])
    ap.add_argument("--m", type=int, nargs="+", default=[1, 16, 64, 256])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import pykrige_b200 as pk

    pts = np.random.default_rng(1).uniform(0.0, 1000.0, size=(2, 1024))
    rows = []
    info = gpu_info()
    print("GPU:", info, flush=True)
    warm = pk.OrdinaryKriging(*data(500, 0)[0].T, data(500, 0)[1], variogram_model="exponential",
                              variogram_parameters=PARAMS)
    warm.execute("points", *pts)
    warm.add_data([1.0], [2.0], [0.5])
    warm.execute("points", *pts)
    del warm
    for N in a.sizes:
        for m in a.m:
            xy, val = data(N, m)
            t_app, t_new, diff = [], [], 0.0
            for _ in range(a.reps):
                base = pk.OrdinaryKriging(xy[:N, 0], xy[:N, 1], val[:N], variogram_model="exponential",
                                          variogram_parameters=PARAMS)
                base.execute("points", *pts)                       # the held factorisation (not timed)
                base._kb_handle.reset_counters()
                t0 = time.perf_counter()
                base.add_data(xy[N:, 0], xy[N:, 1], val[N:])
                za, sa = base.execute("points", *pts)
                t_app.append(time.perf_counter() - t0)
                timings = base._kb_handle.timings()
                del base
                gc.collect()
                t0 = time.perf_counter()
                new = pk.OrdinaryKriging(xy[:, 0], xy[:, 1], val, variogram_model="exponential",
                                         variogram_parameters=PARAMS)
                zn, sn = new.execute("points", *pts)
                t_new.append(time.perf_counter() - t0)
                del new
                gc.collect()
                diff = max(diff, np.abs(za - zn).max() / np.abs(zn).max(), np.abs(sa - sn).max() / np.abs(sn).max())
            row = dict(N=N, m=m, add_data_execute_ms=1e3 * float(np.median(t_app)),
                       new_object_execute_ms=1e3 * float(np.median(t_new)),
                       speedup=float(np.median(t_new) / np.median(t_app)), max_rel_diff=float(diff),
                       append_samples_ms=[1e3 * t for t in t_app], new_samples_ms=[1e3 * t for t in t_new],
                       last_append_handle_timings=timings)
            rows.append(row)
            print(json.dumps({k: row[k] for k in ("N", "m", "add_data_execute_ms", "new_object_execute_ms", "speedup",
                                                  "max_rel_diff")}), flush=True)
    out = dict(gpu=info, points=pts.shape[1], variogram=PARAMS, rows=rows)
    print(json.dumps(out), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
