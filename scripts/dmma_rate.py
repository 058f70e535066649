"""Steady-state fp64 tensor-core (DMMA) rate of the four mma.sync f64 shapes on this GPU.

    python scripts/dmma_rate.py [--iters N] [--json PATH]
    python scripts/dmma_rate.py --sustain SECONDS [--json PATH]

--sustain runs one phase-M stage of the fp64 solve kernel (A / B fragments of two m-tiles and eight n-tiles read from
shared memory each stage) on every SM for about SECONDS each, once with four m16n8k4 and once with one m16n8k16 per
(m-tile, n-tile), and reports the board energy NVML counts over the launch, the median power and SM clock sampled
during it, FMA/clk/SM and the energy per FMA (whole board: static power included).

Loads scripts/libdmma_rate.so (built by `make -C pykrige_b200/csrc`) and, for m8n8k4, m16n8k4, m16n8k8 and m16n8k16 at
1, 2 and 4 warps per SM sub-partition, runs one CTA per SM in which every warp issues 8 independent MMAs per iteration.
Prints FMA/clk/SM (from the per-CTA clock64 cycles), TFLOP/s (from CUDA events) and the SM clock those imply, then each
16x8xK shape's best rate relative to m8n8k4's best. The card name and power limit are read in the same call."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "libdmma_rate.so")
SHAPES = ["m8n8k4", "m16n8k4", "m16n8k8", "m16n8k16"]


def load():
    if not os.path.exists(LIB):
        raise SystemExit("%s is not built: run make -C pykrige_b200/csrc" % LIB)
    lib = ctypes.CDLL(LIB)
    lib.dmma_rate_run.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_float),
                                  ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(ctypes.c_int),
                                  ctypes.POINTER(ctypes.c_longlong)]
    lib.dmma_frag_run.argtypes = [ctypes.c_int] + [ctypes.c_void_p] * 4
    lib.dmma_shape_fmas.restype = ctypes.c_longlong
    lib.dmma_stage_run.argtypes = [ctypes.c_int, ctypes.c_longlong, ctypes.POINTER(ctypes.c_float),
                                   ctypes.POINTER(ctypes.c_longlong)]
    return lib


def stage(lib, k, iters):
    ms, fmas = ctypes.c_float(), ctypes.c_longlong()
    err = lib.dmma_stage_run(k, iters, ctypes.byref(ms), ctypes.byref(fmas))
    if err:
        raise SystemExit("dmma_stage_run(k=%d): cudaError %d" % (k, err))
    return ms.value, fmas.value


def sustain(lib, seconds):
    """Energy per FMA of the phase-M stage with m16n8k4 and m16n8k16, each run for about `seconds`."""
    import threading
    import time
    import pynvml as nv
    nv.nvmlInit()
    dev = nv.nvmlDeviceGetHandleByIndex(0)
    sms = None
    rows = []
    for k in (4, 16):
        ms, _ = stage(lib, k, 20000)                                   # warm-up and calibration
        iters = max(1, int(20000 * seconds * 1e3 / ms))
        samples, stop = [], threading.Event()

        def sample():
            while not stop.is_set():
                samples.append((nv.nvmlDeviceGetPowerUsage(dev) / 1e3, nv.nvmlDeviceGetClockInfo(dev, nv.NVML_CLOCK_SM)))
                time.sleep(0.1)
        th = threading.Thread(target=sample, daemon=True)
        e0 = nv.nvmlDeviceGetTotalEnergyConsumption(dev)               # mJ
        th.start()
        ms, fmas = stage(lib, k, iters)
        stop.set()
        th.join()
        e1 = nv.nvmlDeviceGetTotalEnergyConsumption(dev)
        warm = samples[len(samples) // 5:] or samples                  # drop the first fifth: the clock settles
        watts = sorted(w for w, _ in warm)[len(warm) // 2]
        mhz = sorted(c for _, c in warm)[len(warm) // 2]
        if sms is None:
            import torch
            sms = torch.cuda.get_device_properties(0).multi_processor_count
        joules = (e1 - e0) / 1e3
        r = dict(shape="m16n8k%d" % k, seconds=ms / 1e3, fmas=fmas, joules=joules, median_w=watts, median_sm_mhz=mhz,
                 fma_per_clk_sm=fmas / (sms * mhz * 1e6 * ms / 1e3), tflops=2.0 * fmas / (ms / 1e3) / 1e12,
                 pj_per_fma=joules / fmas * 1e12)
        rows.append(r)
        print("%-9s %.1f s  %.1f J  median %.0f W  SM clock %.0f MHz  %.1f FMA/clk/SM  %.2f TFLOP/s  %.2f pJ/FMA" % (
            r["shape"], r["seconds"], r["joules"], r["median_w"], r["median_sm_mhz"], r["fma_per_clk_sm"], r["tflops"],
            r["pj_per_fma"]), flush=True)
    print("energy per FMA, m16n8k16 / m16n8k4: %.3f" % (rows[1]["pj_per_fma"] / rows[0]["pj_per_fma"]), flush=True)
    return rows


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), (v.strip() for v in out.split(","))))
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


def run(lib, shape, wps, iters):
    ms, sms, fmas = ctypes.c_float(), ctypes.c_int(), ctypes.c_longlong()
    cyc = (ctypes.c_longlong * 1024)()
    err = lib.dmma_rate_run(shape, wps, iters, ctypes.byref(ms), cyc, ctypes.byref(sms), ctypes.byref(fmas))
    if err:
        raise SystemExit("dmma_rate_run(%s, %d): cudaError %d" % (SHAPES[shape], wps, err))
    n = sms.value
    mean_cyc = sum(cyc[i] for i in range(n)) / n
    return dict(shape=SHAPES[shape], warps_per_smsp=wps, ms=ms.value, cycles=mean_cyc,
                fma_per_clk_sm=fmas.value / mean_cyc, tflops=2.0 * fmas.value * n / (ms.value * 1e-3) / 1e12,
                sm_mhz=mean_cyc / (ms.value * 1e3), sms=n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200000)
    ap.add_argument("--json", default=None)
    ap.add_argument("--sustain", type=float, default=None, metavar="SECONDS")
    a = ap.parse_args()
    lib = load()
    info = card()
    print("card:", info, flush=True)
    if a.sustain is not None:
        out = dict(card=info, sustain=sustain(lib, a.sustain), card_after=card())
        if a.json:
            os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
            with open(a.json, "w") as f:
                json.dump(out, f, indent=1)
        return out
    rows = []
    for shape in range(4):
        # iterations scaled so that every shape does about the same FMAs per warp
        it = max(1, a.iters * 256 // lib.dmma_shape_fmas(shape))
        for wps in (1, 2, 4):
            run(lib, shape, wps, max(1, it // 20))             # warm-up (module load, clocks)
            r = min((run(lib, shape, wps, it) for _ in range(3)), key=lambda r: r["cycles"])
            rows.append(r)
            print("%-9s %d warp/SMSP  %7.1f FMA/clk/SM  %6.2f TFLOP/s  (%.2f ms, SM clock %.0f MHz)" % (
                r["shape"], wps, r["fma_per_clk_sm"], r["tflops"], r["ms"], r["sm_mhz"]), flush=True)
    best = {s: max(r["fma_per_clk_sm"] for r in rows if r["shape"] == s) for s in SHAPES}
    ratio = {s: best[s] / best["m8n8k4"] for s in SHAPES}
    print("best FMA/clk/SM:", {s: round(v, 1) for s, v in best.items()})
    print("relative to m8n8k4:", {s: round(v, 2) for s, v in ratio.items()})
    info_after = card()
    out = dict(card=info, card_after=info_after, rows=rows, best_fma_per_clk_sm=best, ratio_to_m8n8k4=ratio)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    return out


if __name__ == "__main__":
    sys.exit(0 if main() else 1)
