"""GPU suite (-m gpu): saved env states on the device (k_save_states, k_load_states) and what the vector env builds on them
(save_states, load_states, load_states_torch): restoring replays a run bit for bit, forks equal their source, a model
mismatch is refused, and neither call synchronises with the host."""
import numpy as np
import pytest

from rig import acts, reset_ended, steady_mt50
from rig import torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode", ["SameStep", "NextStep", "Disabled"])
def test_restore_replays_bitwise(torch_cuda, mode):
    """MT50 @ 4096 in steady state: save, 60 steps with autoresets (DISABLED: the ended envs reset with reset_torch(mask)),
    restore, the same 60 steps again: every output tensor and the final state records are bitwise equal."""
    torch = torch_cuda
    env = steady_mt50(torch, mode)
    rng = np.random.default_rng(5)
    A = [acts(torch, rng, env.num_envs, env.device) for _ in range(60)]

    def run():
        outs = []
        for a in A:
            out = [x.clone() for x in env.step_torch(a)]
            outs.append(out + [reset_ended(env, out)])
        return outs, env.engine.get_state()

    states = env.save_states()
    ref, st_ref = run()
    env.load_states_torch(states)
    got, st_got = run()
    assert sum(int(o[3].sum()) for o in ref) > 100                 # truncations inside the window
    for t, (a, b) in enumerate(zip(ref, got)):
        for x, y in zip(a, b):
            assert (x is None and y is None) or torch.equal(x, y), (mode, t)
    assert st_ref.tobytes() == st_got.tobytes()
    assert not env.engine.faults().any()
    env.close()


def test_forks_equal_their_source(torch_cuda):
    """MT10 with 64 envs per task, driven apart by different actions; every env is forked from its task's first env,
    then one action sequence per task follows: every env equals its source bitwise up to and including the step that
    ends the episode (on that step the terminal observation, which SAME_STEP reports in final_obs: the restart draws
    each env's own next task)."""
    torch = torch_cuda
    from metaworld_b200.vector_env import make_mt_envs
    n, M, k = 640, 40, 15
    env = make_mt_envs("MT10", seed=4, num_envs=n, max_episode_steps=M)
    dev = env.device
    env.reset_torch()
    rng = np.random.default_rng(3)
    for _ in range(k):
        env.step_torch(acts(torch, rng, n, dev))
    src = torch.arange(n, device=dev) % 10                          # env e has task e % 10; its first env is e % 10
    qpos = env.engine.get_state()["qpos"]
    assert not np.array_equal(qpos[10], qpos[0])
    obs = env.load_states_torch(env.save_states(), src=src)
    assert torch.equal(obs, obs[src])
    ended_at = None
    for t in range(k, M + 2):
        out = env.step_torch(acts(torch, rng, 10, dev)[src].contiguous())
        end = bool(out[3][0])
        for x in (env.d_final_obs,) + tuple(out[1:]) if end else out:
            assert torch.equal(x, x[src]), t
        if end:
            ended_at = t
            break
    assert ended_at == M - 1
    assert not env.engine.faults().any() and env.engine.counters()["contacts_dropped"] == 0
    env.close()


def test_numpy_save_and_load_replay(torch_cuda):
    """The numpy API: save between `step`s, run on, load, repeat the actions: observations, rewards, flags, infos (with
    final_info's episode statistics) and curr_path_length are those of the original run."""
    from metaworld_b200.vector_env import make_mt_envs
    n = 50
    env = make_mt_envs("MT10", seed=6, num_envs=n, max_episode_steps=12, num_goals=1)
    env.reset()
    rng = np.random.default_rng(8)
    A = rng.uniform(-1, 1, size=(30, n, 4)).astype(np.float32)
    for a in A[:7]:
        env.step(a)
    st = env.save_states()

    def run():
        outs = [env.step(a) for a in A[7:]]
        return outs, env.get_attr("curr_path_length")

    ref, len_ref = run()
    env.load_states(st)
    got, len_got = run()
    assert any("final_info" in o[4] for o in ref)
    for t, (a, b) in enumerate(zip(ref, got)):
        for x, y in zip(a[:4], b[:4]):
            assert np.array_equal(x, y), t
        assert a[4].keys() == b[4].keys(), t
        for key in a[4]:
            if key == "final_info":
                fa, fb = a[4][key], b[4][key]
                assert all(np.array_equal(fa[i], fb[i]) for i in fa if i != "episode"), t
                assert all(np.array_equal(fa["episode"][i], fb["episode"][i]) for i in fa["episode"]), t
            elif key == "final_obs":
                assert all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(a[4][key], b[4][key])), t
            else:
                assert np.array_equal(a[4][key], b[4][key]), (t, key)
    assert len_ref == len_got
    env.close()


def test_optional_wrappers_restore_bitwise(torch_cuda):
    """normalize_observations, the gymnasium reward normalisation and recurrent_info_in_obs: restoring replays bitwise."""
    torch = torch_cuda
    from metaworld_b200.vector_env import make_mt_envs
    n = 700
    env = make_mt_envs("MT10", seed=2, num_envs=n, max_episode_steps=25, normalize_observations=True,
                       reward_normalization_method="gymnasium", recurrent_info_in_obs=True)
    env.reset_torch()
    rng = np.random.default_rng(1)
    A = [acts(torch, rng, n, env.device) for _ in range(40)]
    for a in A[:10]:
        env.step_torch(a)
    states = env.save_states()

    def run():
        return [[x.clone() for x in env.step_torch(a)] for a in A[10:]]

    ref = run()
    env.load_states_torch(states)
    got = run()
    for t, (a, b) in enumerate(zip(ref, got)):
        assert all(torch.equal(x, y) for x, y in zip(a, b)), t
    env.close()


def test_model_mismatch_is_refused(torch_cuda):
    """The numpy form raises ValueError and leaves every record as it was; the torch form leaves exactly the mismatched
    envs unchanged, loads the others and flags exactly the mismatched envs with fault bit 32.  The C entry points
    reject NULL buffers and n_records < 0."""
    torch = torch_cuda
    from metaworld_b200 import engine as E
    from metaworld_b200.vector_env import make_mt_envs
    n = 100
    env = make_mt_envs("MT10", seed=3, num_envs=n)
    dev = env.device
    env.reset_torch()
    rng = np.random.default_rng(4)
    env.step_torch(acts(torch, rng, n, dev))
    states = env.save_states()
    for _ in range(3):
        env.step_torch(acts(torch, rng, n, dev))
    before = env.engine.get_state()
    src = np.arange(n)
    src[[3, 50]] = [4, 61]                                          # another task
    with pytest.raises(ValueError):
        env.load_states(states, src=src)
    assert env.engine.get_state().tobytes() == before.tobytes()
    env.load_states_torch(states, src=torch.from_numpy(src).to(dev))
    after = env.engine.get_state()
    saved = states.records.cpu().numpy().view(E.ENVSTATE_DTYPE).reshape(-1)
    bad = np.isin(np.arange(n), [3, 50])
    assert after[bad].tobytes() == before[bad].tobytes() and after[~bad].tobytes() == saved[~bad].tobytes()
    f = env.engine.faults()
    assert np.array_equal(f, np.where(bad, 32, 0))
    env.load_states_torch(states, src=torch.from_numpy(src).to(dev))
    with pytest.raises(ValueError):
        env.engine.raise_on_faults()
    L, h, p = E.lib(), env.engine.h, states.records.data_ptr()
    assert L.mw_load_states(h, None, None, -1, p, states.model.data_ptr(), states.hints.data_ptr(), None) == -2
    assert L.mw_save_states(h, None, p, None, states.hints.data_ptr(), None) == -2
    env.close()


def test_save_and_load_do_not_synchronise(torch_cuda):
    """NEXT_STEP with the observation normalisation, after step_torch: save_states and load_states_torch (identity and a
    permutation) run under torch.cuda.set_sync_debug_mode("error")."""
    torch = torch_cuda
    from metaworld_b200.vector_env import make_mt_envs
    n = 100
    env = make_mt_envs("MT10", seed=1, num_envs=n, max_episode_steps=5, autoreset_mode="NextStep", normalize_observations=True)
    dev = env.device
    env.reset_torch()
    rng = np.random.default_rng(0)
    A = [acts(torch, rng, n, dev) for _ in range(6)]
    src = torch.roll(torch.arange(n, device=dev), 10)
    mask = torch.arange(n, device=dev) % 2 == 0
    for a in A:
        env.step_torch(a)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        states = env.save_states()
        env.load_states_torch(states)
        env.load_states_torch(states, env_mask=mask, src=src)
        env.step_torch(A[0])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert not env.engine.faults().any()
    env.close()


@pytest.mark.parametrize("task", ["peg-unplug-side-v3", "box-close-v3"])
def test_forks_taken_in_contact_stay_equal(torch_cuda, task):
    """64 envs of a contact-heavy task run their scripted expert (grasping the plug / the lid) with noise; forked from env
    0 while it is in contact, every env equals env 0 bitwise through 40 more expert steps, and no contact is dropped."""
    torch = torch_cuda
    from metaworld_b200 import benchmarks as B
    from metaworld_b200.vector_env import MetaWorldVecEnv
    n = 64
    env = MetaWorldVecEnv([task] * n, [B.MT1(task, seed=0).train_tasks[:1]] * n, seed=0)
    dev = env.device
    env.reset_torch()
    g = torch.Generator(device=dev).manual_seed(0)
    for _ in range(60):
        a = env.expert_actions_torch() + 0.1 * torch.randn(n, 4, device=dev, generator=g)
        env.step_torch(a.clamp(-1, 1).contiguous())
    _, _, meta = env.engine.debug_forward()
    assert meta[0, 0] > 0                                            # env 0 is in contact at the fork
    print(task, "contacts at the fork:", int(meta[0, 0]), "touching:", bool(env.query_torch(touching=True)["touching"][0]))
    src = torch.zeros(n, dtype=torch.long, device=dev)
    env.load_states_torch(env.save_states(), src=src)
    for t in range(40):
        out = env.step_torch(env.expert_actions_torch())
        for x in out:
            assert torch.equal(x, x[:1].expand_as(x)), t
    assert not env.engine.faults().any() and env.engine.counters()["contacts_dropped"] == 0
    env.close()
