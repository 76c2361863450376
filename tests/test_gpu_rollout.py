"""GPU suite (-m gpu): open-loop rollouts on the device (k_rollout) and what the vector env builds on them (rollout_torch,
rollout): every live row equals fork-and-step (load_states_torch, then step_torch) bit for bit, rows end where the
episode ends, the envs are left untouched in every autoreset mode, and the torch form never synchronises."""
import numpy as np
import pytest

from rig import reset_ended, steady_mt50
from rig import torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu


def _fork_and_step(env, st, A, r):
    """For each candidate k: load `st`, step_torch A[k, h] for every h; every row live at step h equals the rollout `r`
    bitwise (reward, the 7 infos, flags, observation), and a row that ended before step h is flag 4 with zero outputs in
    `r`.  Drains the fault bits of the steps taken after an episode's end (DISABLED: 16).  -> rows that ended in the
    horizon, per candidate"""
    torch = env.torch
    K, H = A.shape[:2]
    ends = []
    for k in range(K):
        env.load_states_torch(st)
        ended = st.ended().clone() if env.autoreset_mode != "SameStep" else torch.zeros(env.num_envs, dtype=torch.bool, device=env.device)
        start = ended.clone()
        for h in range(H):
            obs, rew, term, trunc, info = env.step_torch(A[k, h])
            live = ~ended
            assert torch.equal(r.ended[k, h], ended), (k, h)
            assert torch.equal(r.reward[k, h][live], rew[live]), (k, h)
            assert torch.equal(r.info[k, h][live], info[live]), (k, h)
            assert torch.equal(r.terminated[k, h][live], term[live].bool()), (k, h)
            assert torch.equal(r.truncated[k, h][live], trunc[live].bool()), (k, h)
            assert torch.equal(r.obs[k, h][live], obs[live, :39]), (k, h)
            assert not r.reward[k, h][ended].any() and not r.info[k, h][ended].any() and not r.obs[k, h][ended].any()
            assert not r.terminated[k, h][ended].any() and not r.truncated[k, h][ended].any()
            ended = ended | term.bool() | trunc.bool()
        ends.append(ended & ~start)
        f = env.engine.faults()
        assert not (f & ~16).any()
    return ends


def test_rollout_equals_fork_and_step_mt50(torch_cuda):
    """MT50 @ 4096 in steady state (DISABLED), K = 2, H = 12, with observations: every live row equals fork-and-step
    bitwise; no row reports a fault or a dropped contact."""
    torch = torch_cuda
    env = steady_mt50(torch, "Disabled")
    N, K, H = env.num_envs, 2, 12
    g = torch.Generator(device=env.device).manual_seed(1)
    A = torch.rand(K, H, N, 4, device=env.device, generator=g) * 2 - 1
    st = env.save_states()
    r = env.rollout_torch(A, obs=True)
    assert not r.faults.any() and not r.contacts_dropped.any()
    ends = _fork_and_step(env, st, A, r)
    assert all(int(x.sum()) > 0 for x in ends)                         # truncations inside the horizon
    env.close()


def test_rollout_episodes_end_inside_the_horizon(torch_cuda):
    """MT10 x 64 with 40-step episodes and terminate_on_success (DISABLED), 20 closed-loop expert steps in.  Candidate 0
    replays open loop what the expert does closed loop from the saved state, candidate 1 is noise; H = 30 covers
    success terminations and truncations.  Every live row equals fork-and-step bitwise."""
    torch = torch_cuda
    from metaworld_b200.vector_env import make_mt_envs
    n, H = 640, 30
    env = make_mt_envs("MT10", seed=9, num_envs=n, max_episode_steps=40, terminate_on_success=True, autoreset_mode="Disabled")
    env.reset_torch()
    for _ in range(20):
        reset_ended(env, env.step_torch(env.expert_actions_torch()))
    st = env.save_states()
    plan = []
    for _ in range(H):
        plan.append(env.expert_actions_torch())
        env.step_torch(plan[-1])
    env.engine.faults()
    g = torch.Generator(device=env.device).manual_seed(2)
    A = torch.stack([torch.stack(plan), torch.rand(H, n, 4, device=env.device, generator=g) * 2 - 1]).contiguous()
    env.load_states_torch(st)
    r = env.rollout_torch(A, obs=True)
    assert not r.faults.any() and not r.contacts_dropped.any()
    assert int(r.terminated[0].sum()) > 0 and int(r.truncated[0].sum()) > 0
    _fork_and_step(env, st, A, r)
    env.close()


@pytest.mark.parametrize("mode", ["SameStep", "NextStep", "Disabled"])
def test_rollout_leaves_the_envs_untouched(torch_cuda, mode):
    """MT50 @ 4096 in steady state: a rollout changes no state record and no hint, raises no fault, drops no contact and
    counts no env step; 20 steps after it equal 20 steps after loading the state saved before it."""
    torch = torch_cuda
    env = steady_mt50(torch, mode)
    N = env.num_envs
    g = torch.Generator(device=env.device).manual_seed(3)
    A = torch.rand(3, 10, N, 4, device=env.device, generator=g) * 2 - 1
    steps = [torch.rand(N, 4, device=env.device, generator=g) * 2 - 1 for _ in range(20)]
    env.engine.faults(); env.engine.counters()
    st = env.save_states()
    before = env.engine.get_state()
    env.rollout_torch(A, obs=True)
    assert env.engine.get_state().tobytes() == before.tobytes()
    assert torch.equal(env.save_states().hints, st.hints)
    assert not env.engine.faults().any()
    c = env.engine.counters()
    assert c["contacts_dropped"] == 0 and c["env_steps"] == 0 and c["launches"] == 3       # save, rollout, save

    def run():
        outs = []
        for a in steps:
            out = [x.clone() for x in env.step_torch(a)]
            outs.append(out + [reset_ended(env, out)])
        return outs, env.engine.get_state()

    ref, st_ref = run()
    env.load_states_torch(st)
    got, st_got = run()
    for t, (a, b) in enumerate(zip(ref, got)):
        for x, y in zip(a, b):
            assert (x is None and y is None) or torch.equal(x, y), (mode, t)
    assert st_ref.tobytes() == st_got.tobytes()
    env.close()


def test_rows_of_ended_envs_are_ended_from_step_0(torch_cuda):
    """NEXT_STEP, MT10 x 30 with 5-step episodes and staggered starts: the rows of the envs that ended in the last step
    carry flag 4 from step 0 with zero outputs; the other rows equal fork-and-step."""
    torch = torch_cuda
    from metaworld_b200.vector_env import make_mt_envs
    n = 300
    env = make_mt_envs("MT10", seed=2, num_envs=n, max_episode_steps=5, autoreset_mode="NextStep")
    dev = env.device
    env.reset_torch()
    g = torch.Generator(device=dev).manual_seed(4)
    env.step_torch(torch.rand(n, 4, device=dev, generator=g) * 2 - 1)
    env.reset_torch(torch.arange(n, device=dev) % 2 == 0)
    for _ in range(4):                                               # the odd envs truncate on the last of these
        env.step_torch(torch.rand(n, 4, device=dev, generator=g) * 2 - 1)
    st = env.save_states()
    ended = st.ended()
    assert ended.any() and not ended.all()
    A = torch.rand(2, 6, n, 4, device=dev, generator=g) * 2 - 1
    r = env.rollout_torch(A, obs=True)
    assert r.ended[:, :, ended].all()
    assert not r.reward[:, :, ended].any() and not r.info[:, :, ended].any() and not r.obs[:, :, ended].any()
    _fork_and_step(env, st, A, r)
    env.close()


def test_rollout_does_not_synchronise_and_numpy_form_equals_it(torch_cuda):
    """After a warm-up call, rollout_torch runs under torch.cuda.set_sync_debug_mode("error"); `rollout` returns the same
    bits as numpy arrays."""
    torch = torch_cuda
    from metaworld_b200.vector_env import make_mt_envs
    n = 100
    env = make_mt_envs("MT10", seed=5, num_envs=n, max_episode_steps=8, normalize_observations=True)
    dev = env.device
    env.reset_torch()
    g = torch.Generator(device=dev).manual_seed(5)
    for _ in range(3):
        env.step_torch(torch.rand(n, 4, device=dev, generator=g) * 2 - 1)
    A = torch.rand(4, 9, n, 4, device=dev, generator=g) * 2 - 1
    env.rollout_torch(A[:2])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        r = env.rollout_torch(A, obs=True)
        r = [None if x is None else x.clone() for x in r]
    finally:
        torch.cuda.set_sync_debug_mode(0)
    h = env.rollout(A.cpu().numpy(), obs=True)
    for x, y in zip(r, h):
        assert isinstance(y, np.ndarray) and np.array_equal(x.cpu().numpy(), y)
    assert h.truncated.any()
    env.close()
