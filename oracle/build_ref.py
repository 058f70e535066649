"""Builds oracle/_ref/: the reference's OWN native twins of the hot path, compiled from the reference's sources at
REF_LIB (read-only; no reference source is copied into the repo):

    lib/cok.pyx               _c_exec_loop (cok.pyx:14-96), _c_exec_loop_moving_window (cok.pyx:98-193)
    lib/variogram_models.pyx  the C variogram table (variogram_models.pyx:5-21)

TEST INFRASTRUCTURE ONLY (same rule as oracle/krige_oracle.py): tests/golden/make_golden.py runs the twins and stores
their outputs in tests/golden/ref_twins.npz, which the tests compare against, so no test needs them; bench.py's
cpu_baseline leg also times them when they are built. Outputs go only into oracle/_ref/ (git-ignored):

    oracle/_ref/build/*.c                       Cython-generated C, deleted again after compilation
    oracle/_ref/pykrige/lib/{cok,variogram_models}.<abi>.so
    oracle/_ref/pykrige/__init__.py, lib/__init__.py   empty package markers written by this script

The package has to be importable as `pykrige.lib.*`: Cython bakes the qualified name of the cimported
module (`from .variogram_models cimport get_variogram_model`, cok.pyx:11) into the extension.

    python oracle/build_ref.py          # no-op when the reference's sources are absent
"""
import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
REF_LIB = "/root/reference/src/pykrige/lib"
OUT = os.path.join(HERE, "_ref")
MODULES = ("variogram_models", "cok")


def built():
    suffix = sysconfig.get_config_var("EXT_SUFFIX")
    return all(os.path.exists(os.path.join(OUT, "pykrige", "lib", m + suffix)) for m in MODULES)


def build(force=False):
    """Returns True when oracle/_ref is usable afterwards."""
    if not os.path.isdir(REF_LIB):
        return built()
    if built() and not force:
        return True
    import numpy
    suffix = sysconfig.get_config_var("EXT_SUFFIX")
    bdir = os.path.join(OUT, "build")
    pdir = os.path.join(OUT, "pykrige", "lib")
    os.makedirs(bdir, exist_ok=True)
    os.makedirs(pdir, exist_ok=True)
    for d in (os.path.join(OUT, "pykrige"), pdir):
        with open(os.path.join(d, "__init__.py"), "w") as f:
            f.write("# package marker written by oracle/build_ref.py (the compiled reference twins live here)\n")
    inc = [sysconfig.get_paths()["include"], numpy.get_include()]
    for m in MODULES:
        c_file = os.path.join(bdir, m + ".c")
        subprocess.check_call([sys.executable, "-m", "cython", "-3", os.path.join(REF_LIB, m + ".pyx"), "-o", c_file])
        cmd = ["gcc", "-O2", "-fPIC", "-shared", "-fno-strict-aliasing", "-w",
               "-DNPY_NO_DEPRECATED_API=NPY_1_7_API_VERSION"]
        cmd += ["-I" + i for i in inc] + [c_file, "-o", os.path.join(pdir, m + suffix)]
        subprocess.check_call(cmd)
        os.remove(c_file)              # the generated C quotes the .pyx lines in comments: keep only the binary
    try:
        os.rmdir(bdir)
    except OSError:
        pass
    return built()


def load():
    """Import the compiled twins (pykrige.lib.cok) from oracle/_ref; None when they are not built or
    another `pykrige` package is already imported in this process."""
    if not built():
        return None
    if "pykrige" in sys.modules and not getattr(sys.modules["pykrige"], "__file__", "").startswith(OUT):
        return None
    sys.path.insert(0, OUT)
    try:
        import importlib
        return importlib.import_module("pykrige.lib.cok")
    except Exception:
        return None
    finally:
        sys.path.remove(OUT)


if __name__ == "__main__":
    ok = build(force="--force" in sys.argv)
    print("oracle/_ref:", "built" if ok else "not available")
