"""fp64 solve kernel, config 2 (N=5000): (1) cost of one round of 64 / 32 / 16-point tiles (KB200_TILE forces one width for a
whole launch) -> the constants KB_TILE_COST_32 / _16 of csrc/api.cu; (2) what the automatic tail-tile split gives for the
125 000 points one of 8 GPUs gets, and for the whole grid."""
import os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases, pykrige_b200 as pk
import torch
SMS = torch.cuda.get_device_properties(0).multi_processor_count
xyz, val = cases.synth_data(1002, 5000, 2)
ok = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="exponential", variogram_parameters=[1.0, 300.0, 0.05])
g = np.linspace(0, 1000, 1000)
h = ok._ensure_problem()

def t(count, reps=2):
    best = 1e30
    for _ in range(reps + 1):
        h.reset_counters()
        h.execute_grid(g, g, None, None, 0, count)
        best = min(best, h.timings()["solve_ms"])
    return best

per_round = {}
for tile in (64, 32, 16):
    os.environ["KB200_TILE"] = str(tile)
    rounds = 6
    ms = t(SMS * tile * rounds)
    per_round[tile] = ms / rounds
    print("tile", tile, "points:", SMS * tile * rounds, "->", round(ms, 3), "ms =", round(ms / rounds, 3), "ms per round", flush=True)
print("cost of a round relative to 64-point tiles: 32 ->", round(per_round[32] / per_round[64], 3), " 16 ->", round(per_round[16] / per_round[64], 3), flush=True)
os.environ["KB200_TILE"] = "64"
a = {c: t(c) for c in (125000, 132608, 1000000)}
os.environ.pop("KB200_TILE")
b = {c: t(c) for c in (125000, 132608, 1000000)}
for c in a:
    print(c, "points: 64-point tiles only", round(a[c], 2), "ms; with the tail launch", round(b[c], 2), "ms", flush=True)
