"""GPU suite (-m gpu): NEXT_STEP and DISABLED autoreset in k_step and the partial reset k_reset_masked.  The episodes they
produce are bitwise the episodes of the default SAME_STEP run: only where each transition is reported changes."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch


def _actions(ep, k):
    """The action of every env as a function of (env, episode, step in episode) only."""
    n = len(ep)
    x = 1.3 * np.arange(n)[:, None] + 2.7 * ep[:, None] + 0.37 * k[:, None] + 1.9 * np.arange(4)[None, :]
    return np.sin(x).astype(np.float32)


def _episodes(mode, sampler, n_calls, n_envs=1050, seed=5):
    """Runs MT50 under `mode` ("device": step_torch / reset_torch with the device sampler, "host": numpy step / reset with
    the host's task streams) and returns, per env, the sequence of what it went through: ("reset", obs) and
    ("step", obs, reward, terminated, truncated, info[7], episode return or None), all as bytes."""
    import torch
    from metaworld_b200.vector_env import make_mt_envs
    env = make_mt_envs("MT50", seed=seed, num_envs=n_envs, max_episode_steps=6, terminate_on_success=True, use_one_hot=True,
                       autoreset_mode=mode)
    N = env.num_envs
    seq = [[] for _ in range(N)]
    ep, k = np.zeros(N, np.int64), np.zeros(N, np.int64)
    ended = np.zeros(N, bool)
    obs = (env.reset_torch().cpu().numpy() if sampler == "device" else env.reset()[0])
    for e in range(N):
        seq[e].append(("reset", obs[e].tobytes()))
    b = lambda x: np.asarray(x, np.float64).tobytes()
    for _ in range(n_calls):
        restarting = ended.copy()
        a = _actions(ep, k)
        if sampler == "device":
            o, r, te, tr, inf = (x.cpu().numpy() for x in env.step_torch(torch.from_numpy(a).to(env.device)))
            te, tr = te != 0, tr != 0
            fobs, finf = env.d_final_obs.cpu().numpy(), env.d_final_info.cpu().numpy()
            inf = np.hstack([inf, finf[:, 7:8]])
        else:
            o, r, te, tr, infos = env.step(a)
            inf = np.zeros((N, 8))
            for i, key in enumerate(("success", "near_object", "grasp_success", "grasp_reward", "in_place_reward", "obj_to_target", "unscaled_reward")):
                if key in infos:
                    inf[:, i] = infos[key]
                if mode == "SameStep" and "final_info" in infos:
                    inf[infos["_final_info"], i] = infos["final_info"][key][infos["_final_info"]]
            epi = (infos["final_info"] if mode == "SameStep" and "final_info" in infos else infos).get("episode")
            if epi is not None:
                inf[:, 7] = epi["r"]
            fobs = np.stack([x if x is not None else np.zeros_like(o[0]) for x in infos["final_obs"]]) if "final_obs" in infos else None
        done = te | tr
        for e in range(N):
            if ended[e]:             # NEXT_STEP restart call (the action was ignored)
                assert r[e] == 0 and not done[e] and not inf[e, :7].any()
                seq[e].append(("reset", o[e].tobytes()))
                ended[e] = False
                continue
            if mode == "SameStep" and done[e]:
                seq[e].append(("step", fobs[e].tobytes(), b(r[e]), bool(te[e]), bool(tr[e]), b(inf[e, :7]), b(inf[e, 7])))
                seq[e].append(("reset", o[e].tobytes()))
            else:
                seq[e].append(("step", o[e].tobytes(), b(r[e]), bool(te[e]), bool(tr[e]), b(inf[e, :7]), b(inf[e, 7]) if done[e] else None))
        k[~restarting] += 1
        ep[done] += 1
        k[done] = 0
        if mode == "NextStep":
            ended |= done
        elif mode == "Disabled" and done.any():
            if sampler == "device":
                o = env.reset_torch(torch.from_numpy(done).to(env.device)).cpu().numpy()
            else:
                o, _ = env.reset(options={"reset_mask": done.copy()})
            for e in np.nonzero(done)[0]:
                seq[e].append(("reset", o[e].tobytes()))
    env.close()
    return seq


@pytest.mark.parametrize("sampler", ["device", "host"])
@pytest.mark.parametrize("mode", ["NextStep", "Disabled"])
def test_autoreset_mode_runs_the_same_episodes_as_same_step(torch_cuda, mode, sampler):
    """MT50 x 1050 envs, 6-step episodes (and earlier successes): each env's stream of reset observations and transitions
    (observation, reward, flags, infos, episode return) under NEXT_STEP / DISABLED + reset_mask is bitwise the SAME_STEP
    one; the reset observations pin the goal sequences."""
    ref = _episodes("SameStep", sampler, 20)
    got = _episodes(mode, sampler, 24)
    n_eps = 0
    for e, (x, y) in enumerate(zip(ref, got)):
        m = min(len(x), len(y))
        assert m >= 20 and x[:m] == y[:m], e
        n_eps += sum(1 for it in x[:m] if it[0] == "reset")
    assert n_eps >= 4 * len(ref)


def test_stepping_an_ended_env_with_autoreset_disabled_is_flagged_and_changes_nothing(torch_cuda):
    torch = torch_cuda
    from metaworld_b200.vector_env import make_mt_envs
    env = make_mt_envs("MT10", seed=2, num_envs=40, max_episode_steps=3, autoreset_mode="Disabled")
    env.reset_torch()
    a = torch.zeros(40, 4, device=env.device)
    a[:20, 0] = 1.0
    for _ in range(2):
        env.step_torch(a)
    st0 = env.engine.get_state()
    env.engine.faults()
    env.step_torch(a)               # the 3rd step truncates every env
    st1 = env.engine.get_state()
    assert (st0["ended"] == 0).all() and (st1["ended"] == 1).all()
    o1, r1 = env.d_obs.clone(), env.d_reward.clone()
    assert not env.engine.faults().any()
    mask = torch.zeros(40, dtype=torch.bool, device=env.device)
    mask[::2] = True
    env.reset_torch(mask)           # the even envs restart; the odd ones stay ended
    st2 = env.engine.get_state()
    assert torch.equal(env.d_obs[1::2], o1[1::2]) and not torch.equal(env.d_obs[::2], o1[::2]) and (st2["ended"][::2] == 0).all()
    assert (st2["episode"][::2] == st1["episode"][::2] + 1).all()
    env.step_torch(a)
    f = env.engine.faults()
    assert (f[1::2] == 16).all() and (f[::2] == 0).all()
    st3 = env.engine.get_state()
    assert st3[1::2].tobytes() == st2[1::2].tobytes()                       # the ended envs' records are untouched
    assert torch.equal(env.d_obs[1::2], o1[1::2]) and torch.equal(env.d_reward[1::2], r1[1::2])
    env.step_torch(a)
    with pytest.raises(ValueError, match="autoreset disabled"):
        env.engine.raise_on_faults()
    env.disable_device_sampler()
    env.reset()
    for _ in range(3):
        env.step(np.zeros((40, 4), np.float32))
    with pytest.raises(AssertionError):          # the numpy path checks on the host, before anything is launched
        env.step(np.zeros((40, 4), np.float32))
    assert not env.engine.faults().any()
    env.close()


def test_step_and_step_torch_agree_exactly_under_next_step_with_wrappers(torch_cuda):
    """Recurrent observation + observation normalisation + gymnasium reward normalisation under NEXT_STEP: the numpy and
    the torch paths give bit-identical outputs, restart calls and a partial reset included."""
    torch = torch_cuda
    from metaworld_b200.vector_env import make_ml_envs
    kw = dict(seed=4, meta_batch_size=20, max_episode_steps=4, autoreset_mode="NextStep", recurrent_info_in_obs=True,
              normalize_observations=True, reward_normalization_method="gymnasium")
    a, b = make_ml_envs("ML10", **kw), make_ml_envs("ML10", **kw)
    oa, _ = a.reset()
    ob = b.reset_torch()
    assert np.array_equal(oa, ob.cpu().numpy())
    rng = np.random.default_rng(0)
    n_restart = 0
    for t in range(15):
        if t == 6:
            m = np.arange(20) % 3 == 0
            oa, _ = a.reset(options={"reset_mask": m})
            ob = b.reset_torch(torch.from_numpy(m).to(b.device))
            assert np.array_equal(oa, ob.cpu().numpy()), t
        act = rng.uniform(-1, 1, size=(20, 4)).astype(np.float32)
        oa, ra, tea, tra, infa = a.step(act)
        ob, rb, teb, trb, _ = b.step_torch(torch.from_numpy(act).to(b.device))
        assert np.array_equal(oa, ob.cpu().numpy()) and np.array_equal(ra, rb.cpu().numpy()), t
        assert np.array_equal(tea, teb.cpu().numpy() != 0) and np.array_equal(tra, trb.cpu().numpy() != 0), t
        if "episode" in infa:
            assert np.array_equal(infa["episode"]["r"], b.d_episode_return_post.cpu().numpy()), t
        n_restart += int("success" in infa and (~infa["_success"]).sum())
    assert n_restart >= 25
    a.close(); b.close()


def test_next_step_checkpoint_between_terminal_step_and_restart_resumes_bitwise(torch_cuda):
    from metaworld_b200.vector_env import make_mt_envs
    kw = dict(seed=11, num_envs=20, max_episode_steps=5, use_one_hot=True, terminate_on_success=True, autoreset_mode="NextStep")
    rng = np.random.default_rng(0)
    A = rng.uniform(-1, 1, size=(30, 20, 4)).astype(np.float32)
    a = make_mt_envs("MT10", **kw)
    a.reset()
    for t in range(5):
        a.step(A[t])                 # the 5th step truncates every env that did not succeed earlier
    assert a._ended.any()
    ck = a.call("get_checkpoint")
    ref = [a.step(A[t]) for t in range(5, 30)]
    b = make_mt_envs("MT10", **kw)
    b.reset()
    b.call("load_checkpoint", list(ck))
    got = [b.step(A[t]) for t in range(5, 30)]
    n_done = 0
    for x, y in zip(ref, got):
        assert all(np.array_equal(u, v) for u, v in zip(x[:4], y[:4])) and set(x[4]) == set(y[4])
        if "episode" in x[4]:
            n_done += int(x[4]["_episode"].sum())
            assert np.array_equal(x[4]["episode"]["r"], y[4]["episode"]["r"]) and np.array_equal(x[4]["episode"]["l"], y[4]["episode"]["l"])
    assert n_done >= 40
    assert [tuple(v) for v in a.get_attr("_last_rand_vec")] == [tuple(v) for v in b.get_attr("_last_rand_vec")]
    a.close(); b.close()
