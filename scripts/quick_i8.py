"""The wgmma kernels (dtype='float64x' / 'float64x5' / 'float64x4' int8 slices, 'float32' 3xTF32) vs the fp64 DMMA
kernel: agreement and solve-kernel rate. Prints one JSON line per problem."""
import os, sys, json
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases, pykrige_b200 as pk

sizes = ((300, 1000, "ok"), (1000, 20000, "uk"), (5000, 400000, "ok"), (10000, 600000, "uk"))
if len(sys.argv) > 1 and sys.argv[1] == "big":
    sizes = ((5000, 1000000, "ok"),)
for n, m, cls in sizes:
    xyz, val = cases.synth_data(1002, n, 2)
    if cls == "ok":
        mdl = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="exponential", variogram_parameters=[1.0, 300.0, 0.05])
    else:
        mdl = pk.UniversalKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="exponential", variogram_parameters=[1.0, 300.0, 0.05],
                                  drift_terms=["regional_linear"])
    rng = np.random.default_rng(1)
    px = np.concatenate([rng.uniform(0, 1000, m), xyz[:8, 0]]); py = np.concatenate([rng.uniform(0, 1000, m), xyz[:8, 1]])
    out = {}
    for dt in ("float64", "float64x", "float64x5", "float64x4", "float32"):
        mdl._kb_key = None
        z, ss = mdl.execute("points", px, py, backend="cuda", dtype=dt)
        h = mdl._kb_handle
        h.reset_counters()
        z, ss = mdl.execute("points", px, py, backend="cuda", dtype=dt)
        out[dt] = (z, ss, h.timings()["solve_ms"])
    z64, s64 = out["float64"][:2]
    line = {"n": n, "m": int(px.size), "class": cls}
    for dt, (z, ss, ms) in out.items():
        line[dt] = {"pts_per_s": px.size / (ms * 1e-3),
                    "max_rel_z_vs_f64": float(np.abs(z - z64).max() / np.abs(z64).max()),
                    "max_rel_ss_vs_f64": float(np.abs(ss - s64).max() / np.abs(s64).max()),
                    "ss_at_hits": [float(v) for v in ss[-2:]]}
    print(json.dumps(line), flush=True)
