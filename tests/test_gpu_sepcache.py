"""Separating-axis hints (mw_collide.cuh sep_hint_test): a general convex pair that the hint left by an earlier pass still
proves apart skips GJK/EPA.  The hint only ever rejects pairs GJK itself would find apart, so a build without it
(-DMW_NO_SEPCACHE) must give the same results bit for bit: per-step digests of obs / reward / info (scripts/gpu_ab.py)
and the final device state, with no dropped contacts.  The hinted build must actually reject pairs, so that the
comparison cannot pass with the hints silently off."""
import pytest

from builds import run_digests, variant_lib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nosep_lib():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return variant_lib("MW_NO_SEPCACHE")


def _check(hinted, plain):
    assert hinted["steps"] == plain["steps"] and hinted["state"] == plain["state"]
    assert hinted["dropped"] == plain["dropped"] == 0
    assert plain["profile"]["n_sep_tested"] == 0
    assert hinted["profile"]["n_sep_rejected"] > 0
    # the same pairs reach the GJK/EPA stage in both builds: the hint decides how they are evaluated, not which
    assert hinted["profile"]["n_convex_pairs"] == plain["profile"]["n_convex_pairs"]


def test_sepcache_mt50_is_bitwise_identical(nosep_lib, tmp_path):
    """MT50 @ 4096 envs, 150 steps."""
    _check(run_digests(tmp_path / "hinted.json"), run_digests(tmp_path / "plain.json", nosep_lib))


def test_sepcache_contact_overflow_path_is_bitwise_identical(nosep_lib, tmp_path):
    """MT10 @ 350 envs with a shared-memory capacity of 6 contacts (MW_SMCON=6), so that nearly every pass also takes the
    global-memory overflow path, with and without hints."""
    a = run_digests(tmp_path / "hinted.json", variant_lib("MW_SMCON=6"), benchmark="MT10", envs=350)
    b = run_digests(tmp_path / "plain.json", variant_lib("MW_SMCON=6", "MW_NO_SEPCACHE"), benchmark="MT10", envs=350)
    assert "shared 6" in a["build"] and "shared 6" in b["build"]
    _check(a, b)
