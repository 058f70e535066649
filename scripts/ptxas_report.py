#!/usr/bin/env python
"""Register / stack / spill report of every kernel (ptxas -v; needs no GPU).

    python scripts/ptxas_report.py > ptxas_resources.md

Compiles each csrc/*.cu for sm_90a with -Xptxas -v (objects go to a temporary directory) and prints, per kernel family,
the range of registers per thread, the stack frame and the spill stores / loads over its template instantiations."""
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pykrige_b200", "csrc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def family(mangled):
    full = subprocess.run(["c++filt", mangled], capture_output=True, text=True).stdout.strip()
    m = re.match(r"(?:void\s+)?([A-Za-z_][A-Za-z0-9_:]*)", full)
    return m.group(1) if m else full


def main():
    fam = collections.defaultdict(list)
    with tempfile.TemporaryDirectory() as tmp:
        for src in sorted(f for f in os.listdir(CSRC) if f.endswith(".cu")):
            err = subprocess.run(["nvcc"] + FLAGS + ["-c", os.path.join(CSRC, src), "-o", os.path.join(tmp, src + ".o")],
                                 capture_output=True, text=True, check=True).stderr
            cur = None
            for ln in err.splitlines():
                m = re.search(r"Compiling entry function '(\S+)'", ln)
                if m:
                    cur = dict(file=src, name=m.group(1), regs=0, stack=0, st=0, ld=0)
                    fam[(src, family(m.group(1)))].append(cur)
                    continue
                if cur is None:
                    continue
                m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ln)
                if m:
                    cur["stack"], cur["st"], cur["ld"] = (int(g) for g in m.groups())
                m = re.search(r"Used (\d+) registers", ln)
                if m:
                    cur["regs"] = int(m.group(1))
    print("# ptxas -v resources of the build (sm_90a, `scripts/ptxas_report.py`)\n")
    print("| file | kernel family | instantiations | registers / thread | stack frame (B) | spill stores (B) | spill loads (B) |")
    print("|---|---|---|---|---|---|---|")

    def rng(vals):
        return str(vals[0]) if min(vals) == max(vals) else "%d – %d" % (min(vals), max(vals))
    for (src, name), ks in sorted(fam.items(), key=lambda kv: (kv[0][0], -max(k["regs"] for k in kv[1]))):
        print("| `%s` | `%s` | %d | %s | %s | %s | %s |" % (
            src, name, len(ks), rng([k["regs"] for k in ks]), rng([k["stack"] for k in ks]),
            rng([k["st"] for k in ks]), rng([k["ld"] for k in ks])))
    spilled = [(s, n) for (s, n), ks in fam.items() if any(k["st"] or k["ld"] for k in ks)]
    print("\nKernels with register spills: %s." % (", ".join("`%s`" % n for _, n in spilled) if spilled else "none"))
    print("A non-zero stack frame without spills is a thread-local array indexed at run time (drift rows of the finalize "
          "step, digit arrays of the int8 slicing), not register pressure.")
    return 0


if __name__ == "__main__":
    sys.exit(main())
