"""CPU-side parity fuzz of the DEVICE narrowphase source (metaworld_b200/csrc/mw_collide.cuh) against the oracle.

The CUDA header is compiled for the host by g++ with the warp collapsed to one emulated lane (tests/devcollide/shim.cpp),
so the exact statements that run on the GPU (analytic pairs, aligned cylinder fast paths, GJK, the EPA expansion loop with
its index-ordered compaction) are exercised here, without a GPU, on identical float64 inputs."""
import ctypes as C
import os

import numpy as np
import pytest

from builds import host_shim

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SHIM = os.path.join(HERE, "devcollide", "libdevcollide.so")
G_PLANE, G_SPHERE, G_CAPSULE, G_CYLINDER, G_BOX, G_MESH = 0, 2, 3, 5, 6, 7


@pytest.fixture(scope="module")
def libs():
    shim = host_shim("devcollide", SHIM, headers=("mw_collide.cuh", "mw_math.cuh"))
    from oracle import mjphys
    mjphys.build()
    return shim, C.CDLL(os.path.join(ROOT, "oracle", "libmjphys.so"))


def _call(fn, dev, t1, p1, m1, s1, v1, t2, p2, m2, s2, v2, margin):
    dp, fp = C.POINTER(C.c_double), C.POINTER(C.c_float)
    out = np.zeros(16 * 7)
    keep = []

    def vert(v):
        if v is None:
            return None, 0
        a = np.ascontiguousarray(v, dtype=np.float32 if dev else np.float64)
        keep.append(a)
        return a.ctypes.data_as(fp if dev else dp), len(a)

    def dbl(x):
        a = np.ascontiguousarray(x, dtype=np.float64)
        keep.append(a)
        return a.ctypes.data_as(dp)
    a1, n1 = vert(v1)
    a2, n2 = vert(v2)
    fn.restype = C.c_int
    n = fn(C.c_int(t1), dbl(p1), dbl(m1), dbl(s1), a1, C.c_int(n1), C.c_int(t2), dbl(p2), dbl(m2), dbl(s2), a2, C.c_int(n2),
           C.c_double(margin), out.ctypes.data_as(dp))
    return out[: 7 * n].reshape(n, 7)


def _rot(rng, small=None):
    ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
    ang = rng.uniform(0, np.pi) if small is None else small
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def _shape(rng, t):
    f32 = lambda x: np.asarray(x, dtype=np.float32).astype(np.float64)     # model sizes / hull vertices are float32 on the device
    if t == G_SPHERE:
        return f32([rng.uniform(0.01, 0.04), 0, 0]), None, 0.04
    if t in (G_CAPSULE, G_CYLINDER):
        s = f32([rng.uniform(0.008, 0.04), rng.uniform(0.01, 0.08), 0])
        return s, None, float(np.hypot(s[0], s[1]) + s[0])
    if t == G_BOX:
        s = f32(rng.uniform(0.01, 0.08, size=3))
        return s, None, float(np.linalg.norm(s))
    from scipy.spatial import ConvexHull
    pts = rng.normal(size=(40, 3)) * rng.uniform(0.01, 0.05, size=3)
    v = f32(pts[ConvexHull(pts).vertices])
    return np.zeros(3), v, float(np.abs(v).max() * 1.8)


def _pose_near(rng, r1, r2, aligned):
    R1 = np.eye(3) if aligned else _rot(rng)
    R2 = (np.eye(3)[:, rng.permutation(3)] * rng.choice([-1, 1], size=3)) if aligned else _rot(rng)
    if np.linalg.det(R2) < 0:
        R2[:, 0] *= -1
    d = rng.normal(size=3); d /= np.linalg.norm(d)
    if aligned and rng.random() < 0.7:
        d = np.eye(3)[rng.integers(3)] * rng.choice([-1, 1]) + rng.normal(size=3) * 0.05
        d /= np.linalg.norm(d)
    return np.zeros(3), R1, d * rng.uniform(0.2, 1.0) * (r1 + r2), R2


@pytest.mark.parametrize("aligned", [False, True])
def test_device_narrowphase_matches_oracle(libs, aligned):
    dev, ora = libs
    rng = np.random.default_rng(7 + aligned)
    types = [G_SPHERE, G_CAPSULE, G_CYLINDER, G_BOX, G_MESH]
    total = hits = bad_count = bad_geom = bad_pos = 0
    for it in range(3000):
        t1, t2 = sorted(rng.choice(types, size=2))
        s1, v1, r1 = _shape(rng, t1)
        s2, v2, r2 = _shape(rng, t2)
        p1, R1, p2, R2 = _pose_near(rng, r1, r2, aligned)
        margin = float(rng.choice([0.0, 0.001, 0.002]))
        a = _call(ora.om_narrowphase_pair, False, t1, p1, R1.flatten(), s1, v1, t2, p2, R2.flatten(), s2, v2, margin)
        b = _call(dev.dev_pair, True, t1, p1, R1.flatten(), s1, v1, t2, p2, R2.flatten(), s2, v2, margin)
        total += 1
        if len(a) == 0 and len(b) == 0:
            continue
        hits += 1
        if len(a) != len(b):
            # a count flip is only acceptable at the activation threshold itself
            d = np.concatenate([a[:, 0], b[:, 0]])
            if np.abs(d - margin).min() > 1e-6:
                bad_count += 1
            continue
        a = a[np.lexsort(a[:, 1:4].round(5).T)]; b = b[np.lexsort(b[:, 1:4].round(5).T)]
        if np.abs(a[:, 0] - b[:, 0]).max() > 2e-6 or np.abs(a[:, 4:] - b[:, 4:]).max() > 1e-4:
            bad_geom += 1
        elif np.abs(a[:, 1:4] - b[:, 1:4]).max() > 1e-5:
            bad_pos += 1
    print(f"aligned={aligned}: {total} pairs, {hits} in contact, count mismatches {bad_count}, dist/normal mismatches {bad_geom}, position-only mismatches {bad_pos}")
    assert hits > 300
    assert bad_count == 0 and bad_geom <= 0.01 * hits and bad_pos <= 0.02 * hits
