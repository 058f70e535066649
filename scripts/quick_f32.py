"""dtype='float32' (wgmma 3xTF32) vs float64 at config-2 and config-4 sizes: agreement and solve-kernel rate."""
import os, sys, json
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases, pykrige_b200 as pk
for n, m, cls in ((300, 1000, "ok"), (5000, 400000, "ok"), (10000, 600000, "uk")):
    xyz, val = cases.synth_data(1004, n, 2)
    kw = dict(variogram_model="exponential", variogram_parameters=[1.0, 300.0, 0.05])
    mdl = (pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, **kw) if cls == "ok" else
           pk.UniversalKriging(xyz[:, 0], xyz[:, 1], val, drift_terms=["regional_linear"], **kw))
    rng = np.random.default_rng(1)
    px = np.concatenate([rng.uniform(0, 1000, m), xyz[:8, 0]]); py = np.concatenate([rng.uniform(0, 1000, m), xyz[:8, 1]])
    out = {}
    for dt in ("float64", "float32"):
        mdl._kb_key = None
        mdl.execute("points", px[:2000], py[:2000], backend="cuda", dtype=dt)
        h = mdl._kb_handle; h.reset_counters()
        z, ss = mdl.execute("points", px, py, backend="cuda", dtype=dt)
        out[dt] = (z, ss, h.timings()["solve_ms"])
    z64, s64 = out["float64"][:2]; z32, s32 = out["float32"][:2]
    print(json.dumps({"n": n, "m": int(px.size), "class": cls, "f64_pts_per_s": px.size / (out["float64"][2] * 1e-3),
                      "f32_pts_per_s": px.size / (out["float32"][2] * 1e-3),
                      "max_rel_z": float(np.abs(z32 - z64).max() / np.abs(z64).max()),
                      "max_rel_ss": float(np.abs(s32 - s64).max() / np.abs(s64).max())}), flush=True)
