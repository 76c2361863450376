"""Lane-parallel kinematics and bias forces (mw_kinematics, mw_rne_bias in metaworld_b200/csrc/mw_physics.cuh): one link
per lane, the parent-dependent chain advanced by tree depth.  The form they replace, every lane computing every link in
index order and lane 0 storing, is still built by -DMW_SERIAL_LINKS, and the two must agree bit for bit: the build has no
multiply-add contraction, so an expression gives the same bits whichever lane evaluates it.

CPU test: the CUDA source is compiled for the host with a 32-lane warp emulated by cooperative fibers
(tests/kinlanes/shim.cpp), once per form, and run on every lowered model at random configurations.  The host's sincos is
not CUDA's, but both forms call the same one; what is checked is that no operand, order or rounding differs.
GPU test: per-step digests of an MT50 rollout and the final device state of the two builds (scripts/gpu_ab.py)."""
import ctypes as C

import numpy as np
import pytest

from builds import host_shim, run_digests, variant_lib

JT_FREE, JT_SLIDE, JT_HINGE = 0, 2, 3


def _models():
    """The distinct lowered models of the 50 tasks, by name of the first task that uses each."""
    from metaworld_b200 import lower, modelzoo
    from metaworld_b200.tasks import TASKS
    seen, out = set(), []
    for name, spec in TASKS.items():
        rec = lower.lower(modelzoo.full_model(spec.xml), spec.movable, spec.frames).rec
        key = rec.tobytes()
        if key not in seen:
            seen.add(key)
            out.append((name, rec))
    return out


def test_link_depths_follow_the_parent_table():
    """`link_depth` / `ndepth` emitted by lower.py: roots at 0, a child one below its parent, parents before children."""
    models = _models()
    assert len(models) >= 30
    for name, r in models:
        nl = int(r["nlink"])
        for l in range(nl):
            p = int(r["link_parent"][l])
            assert p < l, name
            assert int(r["link_depth"][l]) == (0 if p < 0 else int(r["link_depth"][p]) + 1), name
        assert int(r["ndepth"]) == int(r["link_depth"][:nl].max()) + 1, name


@pytest.fixture(scope="module")
def shims(tmp_path_factory):
    from metaworld_b200 import build as B
    B.write_header()
    out = tmp_path_factory.mktemp("kinlanes")
    libs = []
    for tag, defs in (("lanes", ()), ("serial", ("MW_SERIAL_LINKS",))):
        lib = host_shim("kinlanes", str(out / f"libkin_{tag}.so"), defs)
        lib.kin_pass.restype = C.c_int
        libs.append(lib)
    return libs


def _pass(lib, rec, qpos, qvel, shift):
    out = np.zeros(8192, dtype=np.uint8)
    model = np.frombuffer(rec.tobytes(), dtype=np.uint8).copy()
    n = lib.kin_pass(model.ctypes.data_as(C.c_void_p), qpos.ctypes.data_as(C.c_void_p), qvel.ctypes.data_as(C.c_void_p),
                     shift.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
    assert 0 < n <= out.size
    return out[:n].tobytes()


def test_lane_parallel_pass_equals_serial_pass_bytewise(shims):
    from metaworld_b200 import lower
    lanes, serial = shims
    rng = np.random.default_rng(11)
    moved = 0
    for name, r in _models():
        nl, nq, nv = int(r["nlink"]), int(r["nq"]), int(r["nv"])
        first = None
        for it in range(200):
            qpos = np.zeros(lower.MAXNQ)
            qpos[:nq] = r["qpos0d"][:nq]
            for l in range(nl):
                jt, qa = int(r["link_jtype"][l]), int(r["link_qadr"][l])
                if jt == JT_FREE:       # any position, a quaternion that is not unit length
                    qpos[qa:qa + 3] = rng.uniform(-1, 1, 3)
                    qpos[qa + 3:qa + 7] = rng.normal(size=4) * rng.uniform(0.2, 3.0)
                elif jt == JT_SLIDE:
                    qpos[qa] += rng.uniform(-0.3, 0.3)
                else:                   # hinge angles well beyond +-pi
                    qpos[qa] += rng.uniform(-12.0, 12.0) if it % 2 else rng.uniform(-1.0, 1.0)
            qvel = np.zeros(lower.MAXDOF)
            qvel[:nv] = rng.normal(size=nv) * 3.0
            shift = rng.uniform(-0.2, 0.2, 3) if it % 3 else np.zeros(3)
            a = _pass(lanes, r, qpos, qvel, shift)
            b = _pass(serial, r, qpos, qvel, shift)
            assert a == b, f"{name}: configuration {it} differs between the lane-parallel and the serial form"
            first = first or a
            moved += a != first
    assert moved > 1000      # the outputs do depend on the inputs: the comparison is not of two constant buffers


@pytest.mark.gpu
def test_serial_links_build_is_bitwise_identical_on_mt50(tmp_path):
    """MT50 @ 4096 envs, 40 random-action steps: the default build against -DMW_SERIAL_LINKS."""
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    a = run_digests(tmp_path / "lanes.json", steps=40)
    b = run_digests(tmp_path / "serial.json", variant_lib("MW_SERIAL_LINKS"), steps=40)
    assert "serial links" in b["build"] and "serial links" not in a["build"]
    assert a["steps"] == b["steps"] and a["state"] == b["state"]
    assert a["dropped"] == b["dropped"] == 0
    assert 0 < a["profile"]["kin"] < b["profile"]["kin"]
