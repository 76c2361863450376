"""Host model of the two-chain Cholesky of csrc/mw_physics.cuh (mw_chol / mw_chol_solve): when the coupling block
A[nb:, :nb] is exactly zero, factoring / back-substituting the two diagonal blocks independently gives, element for element
and bit for bit, what the single right-looking chain gives - the skipped work is exclusively `x -= l * 0`.  The model uses
the kernel's operation order in float32 (numpy has no fused multiply-add: the statement is about dense vs block order within
one arithmetic, which is what the device relies on).  On the GPU, the default build and one built with -DMW_CHOL_ONE_CHAIN
(never split the factorisation) give equal per-step digests of an MT50 rollout and an equal final state (scripts/gpu_ab.py).
"Equal" is up to the sign of zero: the single chain's `x - l * 0`, which the two chains skip, can change the sign of a zero
x, so some warm-start entries of the final state are -0.0 in one build and +0.0 in the other; no later operation can tell
them apart."""
import numpy as np
import pytest

from builds import run_digests, variant_lib

f32 = np.float32


def chol_rows(A, lo, hi):
    """right-looking Cholesky of A[lo:hi, lo:hi] in place (lower triangle), the kernel's order: column j is scaled, then
    subtracted from the trailing columns k = j + 1 ... in increasing k"""
    for j in range(lo, hi):
        piv = f32(np.sqrt(max(A[j, j], f32(1e-30))))
        A[j, j] = piv
        for i in range(j + 1, hi):
            A[i, j] = f32(A[i, j] / piv) if A[i, j] != 0 else A[i, j]
        for k in range(j + 1, hi):
            for i in range(k, hi):
                A[i, k] = f32(A[i, k] - f32(A[i, j] * A[k, j]))


def solve_rows(L, b, lo, hi):
    y = b.copy()
    for j in range(lo, hi):
        xj = f32(y[j] / L[j, j]) if y[j] != 0 else y[j]
        y[j] = xj
        for i in range(j + 1, hi):
            y[i] = f32(y[i] - f32(L[i, j] * xj))
    for j in range(hi - 1, lo - 1, -1):
        xj = f32(y[j] / L[j, j]) if y[j] != 0 else y[j]
        y[j] = xj
        for i in range(lo, j):
            y[i] = f32(y[i] - f32(L[j, i] * xj))
    return y


def spd(rng, n):
    B = rng.normal(size=(n, n))
    return (B @ B.T + n * np.eye(n)).astype(f32)


@pytest.mark.parametrize("nv,nb", [(15, 9), (10, 9), (11, 9), (16, 6), (16, 9), (17, 9)])
def test_two_chains_equal_one_chain(nv, nb):
    rng = np.random.default_rng(nv * 100 + nb)
    for trial in range(20):
        A = np.zeros((nv, nv), dtype=f32)
        A[:nb, :nb] = spd(rng, nb); A[nb:, nb:] = spd(rng, nv - nb)
        if trial % 3 == 0 and nv - nb >= 2:       # structural zeros inside a block (a free body's translational 3 x 3 block is diagonal)
            A[nb + 1, nb] = A[nb, nb + 1] = 0
        b = rng.normal(size=nv).astype(f32)
        if trial % 2 == 0:
            b[nb:] = 0                           # a resting object: exact zeros on the right-hand side
        one = A.copy(); chol_rows(one, 0, nv)
        two = A.copy(); chol_rows(two, 0, nb); chol_rows(two, nb, nv)
        assert np.array_equal(np.tril(one), np.tril(two))
        x1 = solve_rows(one, b, 0, nv)
        x2 = b.copy(); x2[:nb] = solve_rows(two, b, 0, nb)[:nb]; x2[nb:] = solve_rows(two, b, nb, nv)[nb:]
        assert np.array_equal(x1, x2)
        # and it is a solution
        Ad = A.astype(np.float64)
        assert np.allclose(Ad @ x1.astype(np.float64), b, atol=5e-4)


def test_coupled_blocks_need_the_single_chain():
    """A non-zero coupling entry (a contact between gripper and object) makes the block factorisation wrong - which is why
    mw_chol inspects the actual block and falls back to one chain."""
    rng = np.random.default_rng(3)
    nv, nb = 15, 9
    A = spd(rng, nv)
    one = A.copy(); chol_rows(one, 0, nv)
    two = A.copy(); chol_rows(two, 0, nb); chol_rows(two, nb, nv)
    assert not np.allclose(np.tril(one)[nb:, nb:], np.tril(two)[nb:, nb:], atol=1e-3)
    coupled = bool(np.any(A[nb:, :nb] != 0))     # the run-time test of mw_chol
    assert coupled


@pytest.mark.gpu
def test_one_chain_cholesky_build_is_bitwise_identical(tmp_path):
    """MT50 @ 4096 envs, 150 random-action steps: the default build (two chains where the coupling block is zero) against
    -DMW_CHOL_ONE_CHAIN."""
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    a = run_digests(tmp_path / "two.json")
    b = run_digests(tmp_path / "one.json", variant_lib("MW_CHOL_ONE_CHAIN"))
    assert "one-chain cholesky" in b["build"] and "one-chain cholesky" not in a["build"]
    assert a["steps"] == b["steps"] and a["state_values"] == b["state_values"]
    assert a["dropped"] == b["dropped"] == 0
