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


def needs_build():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS + ["mw_model.h", "mw_task_ids.h"]] + [os.path.join(_HERE, "lower.py"), os.path.join(_HERE, "tasks.py"),
            os.path.join(_HERE, "..", "include", "metaworld_b200.h")]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, real_double=False, extra=()):
    write_header()
    if real_double:
        return _build_f64(force, verbose)
    if not force and not needs_build():
        return SO
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_TARGET + ["-O3", "-lineinfo", "-std=c++17", "--use_fast_math" if False else "-DMW_NO_FASTMATH",
           "-Xcompiler", "-fPIC", "-shared", "-o", SO] + [os.path.join(CSRC, s) for s in SOURCES]
    if real_double:
        cmd.insert(1, "-DMW_REAL_DOUBLE")
    if verbose:
        cmd[1:1] = ["-Xptxas", "-v"]
    cmd[1:1] = list(extra)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed")
    if verbose:
        print(r.stdout + r.stderr)
    return SO


def _build_f64(force=False, verbose=False):
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS + ["mw_model.h", "mw_task_ids.h"]] + [os.path.join(_HERE, "..", "include", "metaworld_b200.h")]
    if not force and os.path.exists(SO_F64) and os.path.getmtime(SO_F64) >= max(os.path.getmtime(d) for d in deps if os.path.exists(d)):
        return SO_F64
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, "-DMW_REAL_DOUBLE", "-DWARPS_PER_BLOCK=3"] + NVCC_TARGET + ["-O3", "-lineinfo", "-std=c++17",
           "-Xcompiler", "-fPIC", "-shared", "-o", SO_F64] + [os.path.join(CSRC, s) for s in SOURCES]
    if verbose:
        cmd[1:1] = ["-Xptxas", "-v"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed (f64 build)")
    if verbose:
        print(r.stdout + r.stderr)
    return SO_F64


def build_variant(path, defines=(), force=False):
    """A build of the float32 engine with extra -D macros (test-only: e.g. MW_SMCON=6 makes almost every env take the
    overflow path, whose results must be bit-identical to the standard build; tests/test_gpu.py).  Returns the library's
    path: `path`, or a file of the same name in a per-user temporary directory when `path`'s directory cannot be written
    (tests may run from a read-only checkout)."""
    write_header()
    try:
        os.makedirs(os.path.dirname(path), exist_ok=True)
        writable = os.access(os.path.dirname(path), os.W_OK)
    except OSError:
        writable = False
    if not writable:
        path = os.path.join(tempfile.gettempdir(), f"metaworld_b200-{os.getuid()}", os.path.basename(path))
        os.makedirs(os.path.dirname(path), exist_ok=True)
    srcs = [os.path.join(CSRC, f) for f in SOURCES + HEADERS + ["mw_model.h", "mw_task_ids.h"]]
    if not force and os.path.exists(path) and os.path.getmtime(path) >= max(os.path.getmtime(d) for d in srcs):
        return path
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + [f"-D{d}" for d in defines] + NVCC_TARGET + ["-O3", "-lineinfo", "-std=c++17", "-DMW_NO_FASTMATH",
                                                  "-Xcompiler", "-fPIC", "-shared", "-o", path] + [os.path.join(CSRC, s) for s in SOURCES]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed (variant build)")
    return path


if __name__ == "__main__":
    if "--double" in sys.argv:
        print(build(force=True, verbose="-v" in sys.argv, real_double=True))
    elif "--single" in sys.argv:
        print(build(force=True, verbose="-v" in sys.argv))
    else:   # both libraries: the float32 step engine and the float64 snapshot builder
        print(build(force=True, verbose="-v" in sys.argv))
        print(_build_f64(True, "-v" in sys.argv))
