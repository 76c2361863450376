"""Builds libmwb200.so (the CUDA engine, C ABI in include/metaworld_b200.h) in-tree with nvcc for sm_90a (H100)."""
from __future__ import annotations

import os
import subprocess
import sys
import tempfile

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
SO = os.path.join(_HERE, "libmwb200.so")
SO_F64 = os.path.join(_HERE, "libmwb200_f64.so")   # same kernels with real=double (parity-analysis build)
SOURCES = ["mw_engine.cu"]
# Hopper only: the kernels use TMA bulk copies with mbarrier completion (cp.async.bulk, sm_90+)
NVCC_TARGET = ["-gencode", "arch=compute_90a,code=sm_90a"]
# No multiply-add contraction at all (front end and ptxas): contraction is a per-build code-generation decision, and on
# sm_90a the shared-memory and the global-overflow instantiations of the constraint code were contracted differently, so
# an env's results depended on where its constraint rows were stored.  Without contraction every build rounds each
# operation exactly as written (DESIGN.md section 4, "Storage-independent results").
NVCC_TARGET += ["--fmad=false"]
HEADERS = ["mw_math.cuh", "mw_collide.cuh", "mw_physics.cuh", "mw_tasks.cuh", "mw_tasks_gen.cuh", "mw_policies.cuh"]
# what every library is rebuilt from: the sources, the generated headers and the generators behind them, the C ABI header
DEPS = [os.path.join(CSRC, f) for f in SOURCES + HEADERS + ["mw_model.h", "mw_task_ids.h"]] + [
    os.path.join(_HERE, "lower.py"), os.path.join(_HERE, "tasks.py"), os.path.join(_HERE, "..", "include", "metaworld_b200.h")]


def write_header():
    from . import lower

    path = os.path.join(CSRC, "mw_model.h")
    txt = lower.emit_header()
    if not os.path.exists(path) or open(path).read() != txt:
        with open(path, "w") as f:
            f.write(txt)
    from . import tasks
    p2 = os.path.join(CSRC, "mw_task_ids.h")
    txt2 = tasks.emit_task_enum()
    if not os.path.exists(p2) or open(p2).read() != txt2:
        with open(p2, "w") as f:
            f.write(txt2)
    return path


def needs_build(path=SO):
    """True when the library at `path` is missing or older than one of DEPS."""
    if not os.path.exists(path):
        return True
    t = os.path.getmtime(path)
    return any(os.path.getmtime(d) > t for d in DEPS)


def _nvcc(path, defines, verbose):
    """Compiles the engine with -D`defines` into `path`."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + (["-Xptxas", "-v"] if verbose else []) + [f"-D{d}" for d in defines] + NVCC_TARGET + [
        "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-o", path] + [os.path.join(CSRC, s) for s in SOURCES]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError(f"nvcc failed ({os.path.basename(path)})")
    if verbose:
        print(r.stdout + r.stderr)
    return path


def _build(path, defines, force, verbose):
    write_header()
    if force or needs_build(path):
        _nvcc(path, defines, verbose)
    return path


def build(force=False, verbose=False, real_double=False):
    if real_double:
        return _build(SO_F64, ["MW_REAL_DOUBLE", "WARPS_PER_BLOCK=3"], force, verbose)
    return _build(SO, [], force, verbose)


def build_variant(path, defines=(), force=False):
    """A build of the float32 engine with extra -D macros (test-only: e.g. MW_SMCON=6 makes almost every env take the
    overflow path, whose results must be bit-identical to the standard build; tests/test_gpu.py).  Returns the library's
    path: `path`, or a file of the same name in a per-user temporary directory when `path`'s directory cannot be written
    (tests may run from a read-only checkout)."""
    try:
        os.makedirs(os.path.dirname(path), exist_ok=True)
        writable = os.access(os.path.dirname(path), os.W_OK)
    except OSError:
        writable = False
    if not writable:
        path = os.path.join(tempfile.gettempdir(), f"metaworld_b200-{os.getuid()}", os.path.basename(path))
        os.makedirs(os.path.dirname(path), exist_ok=True)
    return _build(path, list(defines), force, False)


if __name__ == "__main__":
    verbose = "-v" in sys.argv
    if "--double" in sys.argv:
        print(build(force=True, verbose=verbose, real_double=True))
    elif "--single" in sys.argv:
        print(build(force=True, verbose=verbose))
    else:   # both libraries: the float32 step engine and the float64 snapshot builder
        print(build(force=True, verbose=verbose))
        print(build(force=True, verbose=verbose, real_double=True))
