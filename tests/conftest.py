import os
import sys

import pytest

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")   # before CUDA is initialised: see groth16_b200/__init__.py
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


def _newest(paths):
    return max((os.path.getmtime(p) for p in paths if os.path.exists(p)), default=0.0)


def _ensure_built():
    """The shared libraries are build artefacts (git-ignored): build them on demand so that a fresh checkout can run the
    CPU tier (ABI symbol check, oracle pinning) without a separate build step, and never test a stale .so silently.

    In a development tree `make` is the staleness check (headers tracked through the -MMD dependency files).  A tree copied
    to a GPU machine with the built libraries but WITHOUT the object files would make `make` recompile everything (minutes
    of nvcc) just to relink the same code, so there the copied library is used as it is when it is at least as new as every
    source it is built from, and rebuilt otherwise."""
    import glob
    import shutil
    import subprocess
    csrc = os.path.join(ROOT, "groth16_b200", "csrc")
    lib = os.path.join(ROOT, "groth16_b200", "libg16b200.so")
    wl = os.path.join(ROOT, "groth16_b200", "libg16workload.so")
    orc = os.path.join(ROOT, "oracle", "liboracle.so")
    jobs = str(max(1, min(16, os.cpu_count() or 1)))
    if shutil.which("g++") or not os.path.exists(orc):
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-j", jobs])
    sources = [p for pat in ("*.cu", "*.cuh", "*.h", "Makefile") for p in glob.glob(os.path.join(csrc, pat))]
    sources += glob.glob(os.path.join(ROOT, "include", "*.h"))
    shipped = (os.path.exists(lib) and os.path.exists(wl) and not glob.glob(os.path.join(csrc, "*.o"))
               and min(os.path.getmtime(lib), os.path.getmtime(wl)) >= _newest(sources))
    if shipped:
        return
    if shutil.which("nvcc") or not os.path.exists(lib):
        subprocess.check_call(["make", "-s", "-C", csrc, "-j", jobs])


_ensure_built()
