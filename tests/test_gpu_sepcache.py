"""Separating-axis hints (mw_collide.cuh sep_hint_test): a general convex pair that the hint left by an earlier pass still
proves apart skips GJK/EPA.  The hint only ever rejects pairs GJK itself would find apart, so a build without it
(-DMW_NO_SEPCACHE) must give the same results bit for bit: per-step digests of obs / reward / info (scripts/gpu_ab.py)
and the final device state, with no dropped contacts.  The hinted build must actually reject pairs, so that the
comparison cannot pass with the hints silently off."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def nosep_lib():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from metaworld_b200 import build as B
    return B.build_variant(os.path.join(ROOT, "tests", "_build", "libmwb200_nosep.so"), ["MW_NO_SEPCACHE"])


def _run(tmp_path, name, lib, args, extra_env=None):
    env = dict(os.environ)
    env.pop("MW_B200_LIB", None); env.pop("MW_B200_SPLIT_FRAC", None)
    if lib:
        env["MW_B200_LIB"] = lib
    env.update(extra_env or {})
    out = str(tmp_path / f"{name}.json")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "gpu_ab.py"), out, *args], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    return json.load(open(out))


def _check(hinted, plain):
    assert hinted["steps"] == plain["steps"] and hinted["state"] == plain["state"]
    assert hinted["dropped"] == plain["dropped"] == 0
    assert plain["profile"]["n_sep_tested"] == 0
    assert hinted["profile"]["n_sep_rejected"] > 0
    # the same pairs reach the GJK/EPA stage in both builds: the hint decides how they are evaluated, not which
    assert hinted["profile"]["n_convex_pairs"] == plain["profile"]["n_convex_pairs"]


def test_sepcache_mt50_is_bitwise_identical(nosep_lib, tmp_path):
    """MT50 @ 4096 envs, 150 steps."""
    _check(_run(tmp_path, "hinted", None, ["150"]), _run(tmp_path, "plain", nosep_lib, ["150"]))


def test_sepcache_contact_overflow_path_is_bitwise_identical(nosep_lib, tmp_path):
    """MT10 @ 350 envs with a shared-memory capacity of 6 contacts (MW_SMCON=6), so that nearly every pass also takes the
    global-memory overflow path, with and without hints."""
    from metaworld_b200 import build as B
    hinted = B.build_variant(os.path.join(ROOT, "tests", "_build", "libmwb200_smcon6.so"), ["MW_SMCON=6"])
    plain = B.build_variant(os.path.join(ROOT, "tests", "_build", "libmwb200_smcon6_nosep.so"), ["MW_SMCON=6", "MW_NO_SEPCACHE"])
    a = _run(tmp_path, "hinted", hinted, ["150", "MT10", "350"])
    b = _run(tmp_path, "plain", plain, ["150", "MT10", "350"])
    assert "shared 6" in a["build"] and "shared 6" in b["build"]
    _check(a, b)
