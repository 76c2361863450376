"""The builds the tests compare: engine variants (`variant_lib`), host builds of device sources (`host_shim`), and the
rollout digests of a build (`run_digests`, scripts/gpu_ab.py)."""
import ctypes as C
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "metaworld_b200", "csrc")
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from gpu_ab import run_digests  # noqa: E402,F401


def variant_lib(*defines):
    """The float32 engine built with -D`defines`, at tests/_build/libmwb200_<tag>.so (MW_SMCON=6, MW_NO_SEPCACHE ->
    libmwb200_smcon6_no_sepcache.so)."""
    from metaworld_b200 import build as B
    tag = "_".join(d.lower().removeprefix("mw_").replace("=", "") for d in defines)
    return B.build_variant(os.path.join(HERE, "_build", f"libmwb200_{tag}.so"), defines)


def host_shim(name, path, defines=(), headers=()):
    """tests/<name>/shim.cpp compiled for the host with -D`defines` into `path`, rebuilt when the shim or one of `headers`
    (files of metaworld_b200/csrc) is newer; loaded with ctypes.  No multiply-add contraction, as nvcc --fmad=false."""
    src = os.path.join(HERE, name, "shim.cpp")
    deps = [src] + [os.path.join(CSRC, h) for h in headers]
    if not os.path.exists(path) or os.path.getmtime(path) < max(os.path.getmtime(d) for d in deps):
        os.makedirs(os.path.dirname(path), exist_ok=True)
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=c++17", "-w", *(f"-D{d}" for d in defines),
                        "-o", path, src], check=True)
    return C.CDLL(path)
