"""fp64 solve kernel, config 2 (N=5000): (1) cost of one round of 64 / 32 / 16-point tiles (KB200_TILE forces one width for a
whole launch) -> the constants KB_TILE_COST_32 / _16 of csrc/api.cu; (2) what the automatic tail-tile split gives for the
125 000 points one of 8 GPUs gets, and for the whole grid.

Beside each round it prints the median SM clock (NVML) during the timed calls and the DMMA-busy fraction that implies:
the FMAs the m16n8k16 MMAs execute / (128 FMA/clk/SM x SMs x clock x solve time). The card name and power limit are
printed first."""
import os, subprocess, sys, threading, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases, pykrige_b200 as pk
import torch
SMS = torch.cuda.get_device_properties(0).multi_processor_count
N = 5000
xyz, val = cases.synth_data(1002, N, 2)
ok = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="exponential", variogram_parameters=[1.0, 300.0, 0.05])
g = np.linspace(0, 1000, 1000)
h = ok._ensure_problem()

q = "name,power.limit,clocks.max.sm"
print("card:", subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip(), flush=True)


def mma_fmas_per_point(n, na=2):
    """FMAs the MMAs of one point execute: each 16-row m-tile of W runs one 16-deep k tile per stage up to its diagonal;
    the m-tiles holding the na dual rows (ordinary kriging: U and zeta) run all of them."""
    nk = (n + 15) // 16
    return sum(16 * 16 * (nk if r0 + 15 >= n else r0 // 16 + 1) for r0 in range(0, n + na, 16))


class Clock(threading.Thread):
    def __init__(self):
        super().__init__(daemon=True)
        self.samples, self.stop = [], False

    def run(self):
        import pynvml as nv
        nv.nvmlInit()
        d = nv.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        while not self.stop:
            self.samples.append(nv.nvmlDeviceGetClockInfo(d, nv.NVML_CLOCK_SM))
            time.sleep(0.05)


def t(count, reps=2):
    best = 1e30
    c = Clock()
    c.start()
    for _ in range(reps + 1):
        h.reset_counters()
        h.execute_grid(g, g, None, None, 0, count)
        best = min(best, h.timings()["solve_ms"])
    c.stop = True
    c.join()
    return best, (float(np.median(c.samples)) if c.samples else float("nan"))

per_round = {}
for tile in (64, 32, 16):
    os.environ["KB200_TILE"] = str(tile)
    rounds = 6
    ms, mhz = t(SMS * tile * rounds)
    per_round[tile] = ms / rounds
    busy = mma_fmas_per_point(N) * SMS * tile * rounds / (128.0 * SMS * mhz * 1e6 * ms * 1e-3)
    print("tile", tile, "points:", SMS * tile * rounds, "->", round(ms, 3), "ms =", round(ms / rounds, 3), "ms per round;",
          "SM clock %.0f MHz, DMMA busy %.3f" % (mhz, busy), flush=True)
print("cost of a round relative to 64-point tiles: 32 ->", round(per_round[32] / per_round[64], 3), " 16 ->", round(per_round[16] / per_round[64], 3), flush=True)
os.environ["KB200_TILE"] = "64"
a = {c: t(c)[0] for c in (125000, 132608, 1000000)}
os.environ.pop("KB200_TILE")
b = {c: t(c)[0] for c in (125000, 132608, 1000000)}
for c in a:
    print(c, "points: 64-point tiles only", round(a[c], 2), "ms; with the tail launch", round(b[c], 2), "ms", flush=True)
