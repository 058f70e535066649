"""Steady-state fp64 tensor-core (DMMA) rate of the four mma.sync f64 shapes on this GPU.

    python scripts/dmma_rate.py [--iters N] [--json PATH]

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
    return lib


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
    a = ap.parse_args()
    lib = load()
    info = card()
    print("card:", info, flush=True)
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
