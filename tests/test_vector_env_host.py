"""Host logic of `MetaWorldVecEnv` (task selection, SAME_STEP autoreset bookkeeping, info dict layout, attribute RPC,
checkpointing) driven with a CPU stand-in for the CUDA engine: the real class, a scripted "engine"."""
import numpy as np
import pytest
import torch

from metaworld_b200 import benchmarks as B
from metaworld_b200.engine import INFO_KEYS
from metaworld_b200.vector_env import MetaWorldVecEnv


class FakeEngine:
    """Keeps per-env (snapshot id, path length); obs[0] = snapshot id, obs[1] = path length; success when path length == 3
    for odd env ids; truncation at max_episode_steps; final_info[7] = episode return = number of steps."""

    def __init__(self, names):
        self.torch = torch
        self.device = torch.device("cpu")
        self.specs = list(names)
        self.n_snap = 0
        self.max_steps, self.tos = 500, False

    def build_snapshots(self, mi, rvs, po):
        ids = np.arange(self.n_snap, self.n_snap + len(mi), dtype=np.int32)
        self.n_snap += len(mi)
        return ids

    def set_envs(self, env_model):
        self.n = len(env_model)
        self.snap = torch.zeros(self.n, dtype=torch.int32)
        self.plen = torch.zeros(self.n)

    def set_options(self, max_steps, tos, seed):
        self.max_steps, self.tos = max_steps, bool(tos)

    def get_state(self):
        from metaworld_b200.engine import ENVSTATE_DTYPE
        st = np.zeros(self.n, dtype=ENVSTATE_DTYPE)
        st["snapshot"] = self.snap.numpy(); st["path_len"] = self.plen.numpy()
        return st

    def set_state(self, st):
        self.snap[:] = torch.from_numpy(st["snapshot"].astype(np.int32)); self.plen[:] = torch.from_numpy(st["path_len"].astype(np.float32))

    def reset(self, snapshot_ids, obs, env_ids=None):
        self.snap[:] = snapshot_ids
        self.plen[:] = 0
        obs[:, :39] = 0
        obs[:, 0] = self.snap.float()

    def step(self, actions, obs, reward, term, trunc, info, final_obs, final_info, next_snapshot):
        self.plen += 1
        succ = (self.plen == 3) & (torch.arange(self.n) % 2 == 1)
        t = succ & self.tos
        tr = self.plen >= self.max_steps
        obs[:, :39] = 0; obs[:, 0] = self.snap.float(); obs[:, 1] = self.plen
        reward[:] = 1.0
        info[:] = 0; info[:, 0] = succ.float()
        term[:] = t.to(torch.uint8); trunc[:] = tr.to(torch.uint8)
        if info.shape[1] >= 9:          # packed record (include/metaworld_b200.h: info_stride >= 9)
            info[:, 7] = reward; info[:, 8] = (t.int() + 2 * tr.int()).float()
        done = t | tr
        final_obs[done] = obs[done]
        final_info[done, :7] = info[done][:, :7]; final_info[done, 7] = self.plen[done]
        self.snap[done] = next_snapshot[done]
        self.plen[done] = 0
        obs[done, 0] = self.snap[done].float(); obs[done, 1] = 0


def make(names, num_envs, **kw):
    tasks_all = B.make_tasks(names, False, seed=1, n_goals=4)
    tasks = [[t for t in tasks_all if t.env_name == n] for n in names]
    return MetaWorldVecEnv(names, tasks, num_envs=num_envs, seed=5, engine=FakeEngine(names), **kw), tasks


def test_reset_step_autoreset_and_info_layout():
    names = ["reach-v3", "push-v3", "door-open-v3"]
    env, tasks = make(names, 6, max_episode_steps=4, use_one_hot=True, num_tasks=3, terminate_on_success=True)
    obs, info = env.reset()
    assert obs.shape == (6, 42) and obs.dtype == np.float32 and info == {}
    assert np.array_equal(obs[:, 39:], np.tile(np.eye(3, dtype=np.float32), (2, 1)))          # env e has type e % 3
    snap0 = obs[:, 0].astype(int)
    for e in range(6):       # the snapshot every env started from belongs to its own task type
        assert env.sub[e].current_task in tasks[e % 3] and snap0[e] == env._snap(env.sub[e].current_task)
    seen_final = 0
    for t in range(1, 9):
        obs, r, term, trunc, info = env.step(np.zeros((6, 4), np.float32))
        assert r.dtype == np.float64 and term.dtype == bool and trunc.dtype == bool
        done = term | trunc
        for k in (INFO_KEYS if not done.all() else ()):      # SAME_STEP: a finished env's step info lives in final_info only
            assert info[k].shape == (6,) and np.array_equal(info["_" + k], ~done) and not info[k][done].any()
        assert ("success" in info) == (not done.all())
        if t == 3:           # odd envs succeed on their 3rd step and terminate (terminate_on_success)
            assert np.array_equal(term, np.arange(6) % 2 == 1)
        if done.any():
            seen_final += 1
            assert np.array_equal(info["_final_obs"], done) and np.array_equal(info["_final_info"], done)
            fi = info["final_info"]
            assert np.array_equal(fi["_episode"], done) and np.array_equal(fi["episode"]["l"][done], fi["episode"]["r"][done].astype(int))
            for e in np.nonzero(done)[0]:
                assert info["final_obs"][e].shape == (42,) and info["final_obs"][e][1] == fi["episode"]["l"][e]
                assert obs[e, 1] == 0 and obs[e, 0] == env._snap(env.sub[e].current_task)     # restarted from its newly selected task
            assert all(info["final_obs"][e] is None for e in np.nonzero(~done)[0])
    assert seen_final >= 3


def test_pseudorandom_task_cycle_and_attribute_rpc():
    names = ["reach-v3", "push-v3"]
    env, tasks = make(names, 2, max_episode_steps=2, task_select="pseudorandom")
    env.reset()
    # PseudoRandomTaskSelectWrapper (wrappers.py:122-160) does not re-sample on reset by default: the task only changes on
    # `sample_tasks`, cycling through a freshly shuffled list every len(tasks) draws
    first = [env.sub[e].current_task for e in range(2)]
    for _ in range(3):
        _, _, term, trunc, _ = env.step(np.zeros((2, 4), np.float32))
    assert [env.sub[e].current_task for e in range(2)] == first
    visited = [[t] for t in first]
    for _ in range(7):
        env.call("sample_tasks")
        for e in range(2):
            visited[e].append(env.sub[e].current_task)
    for e in range(2):
        v = visited[e]
        assert sorted(map(id, v[:4])) == sorted(map(id, tasks[e])) and sorted(map(id, v[4:8])) == sorted(map(id, tasks[e]))
    assert env.get_attr("task_name") == ("reach-v3", "push-v3")
    assert env.get_attr("terminate_on_success") == (False, False)
    env.call("toggle_terminate_on_success", True)
    assert env.get_attr("terminate_on_success") == (True, True) and env.engine.tos
    env.set_attr("terminate_on_success", False)
    assert not env.engine.tos
    rv = env.get_attr("_last_rand_vec")
    assert len(rv) == 2 and len(rv[0]) == 6
    with pytest.raises(AttributeError):
        env.get_attr("no_such_attribute")


def test_optional_wrappers_keep_one_state_across_numpy_and_torch_paths():
    """The optional wrappers' statistics are shared by `step` and `step_torch`: reset_torch() returns the uploaded output of
    reset(), so the observation statistics count the reset observation once, and a run that alternates the two step paths
    follows the all-numpy run up to torch's CPU `sqrt` rounding."""
    kw = dict(max_episode_steps=3, task_select="pseudorandom", use_one_hot=True, num_tasks=2, recurrent_info_in_obs=True,
              reward_normalization_method="gymnasium", normalize_observations=True)
    a, _ = make(["reach-v3", "push-v3"], 4, **kw)
    b, _ = make(["reach-v3", "push-v3"], 4, **kw)
    oa, _ = a.reset()
    ob = b.reset_torch()
    assert np.array_equal(oa, ob.numpy()) and np.array_equal(np.asarray(b.post.obs_count), np.full((4, 1), 1 + 1e-4))
    rng = np.random.default_rng(0)
    n_done = 0
    for t in range(10):
        act = rng.uniform(-1, 1, size=(4, 4)).astype(np.float32)
        obs, rew, term, trunc, info = a.step(act)
        done = term | trunc
        if t % 2:
            o2, r2, term2, trunc2, info2 = b.step(act)
            fo2 = np.stack([info2["final_obs"][e] for e in np.nonzero(done)[0]]) if done.any() else None
            ep2 = info2["final_info"]["episode"]["r"] if done.any() else None
        else:
            o2, r2, term2, trunc2, _ = (x.numpy() for x in b.step_torch(torch.from_numpy(act)))
            fo2, ep2 = b.d_final_obs_post.numpy()[done], np.asarray(b.d_episode_return_post)
        assert np.array_equal(term, term2 != 0) and np.array_equal(trunc, trunc2 != 0)
        np.testing.assert_allclose(o2, obs, rtol=1e-6, atol=0)
        np.testing.assert_allclose(r2, rew, rtol=1e-6, atol=0)
        if done.any():
            n_done += int(done.sum())
            np.testing.assert_allclose(fo2, np.stack([info["final_obs"][e] for e in np.nonzero(done)[0]]), rtol=1e-6, atol=0)
            np.testing.assert_allclose(ep2, info["final_info"]["episode"]["r"], rtol=1e-6, atol=0)
    assert n_done >= 8


def test_checkpoint_round_trip_restores_task_stream():
    """Reference format (metaworld/wrappers.py:125-142,275-322): (env_id, dict) per sub-env; a second env that loads it
    continues with the same task sequence (cross-checked against the reference itself in tests/test_refpin_vector.py)."""
    names = ["reach-v3", "push-v3"]
    env, _ = make(names, 4, max_episode_steps=2)
    env.reset()
    env.step(np.zeros((4, 4), np.float32))
    ck = env.call("get_checkpoint")
    assert len(ck) == 4 and all(isinstance(c, tuple) and len(c) == 2 for c in ck)
    assert ck[0][0] == "<class 'metaworld.envs.sawyer_reach_v3.SawyerReachEnvV3'>_0" and ck[1][0].endswith("SawyerPushEnvV3'>_1")
    assert set(ck[0][1]) >= {"tasks", "rng_state", "sample_tasks_on_reset", "env_rng_state"}
    assert set(ck[0][1]["env_rng_state"]) == {"np_random_state", "action_space_rng_state", "obs_space_rng_state", "goal_space_rng_state"}
    assert isinstance(ck[0][1]["tasks"][0]["data"], str)          # base64, json-serialisable
    import json
    json.dumps([c[1]["tasks"] for c in ck])
    a = []
    for _ in range(8):
        o, *_ = env.step(np.zeros((4, 4), np.float32)); a.append(o[:, 0].copy())
    env2, _ = make(names, 4, max_episode_steps=2)
    env2.reset()
    env2.step(np.zeros((4, 4), np.float32))
    env2.call("load_checkpoint", list(reversed(ck)))      # matched by env_id, not by position
    b = []
    for _ in range(8):
        o, *_ = env2.step(np.zeros((4, 4), np.float32)); b.append(o[:, 0].copy())
    # FakeEngine's obs[0] is the snapshot id each env runs: the restored sampler reproduces the task sequence
    assert np.array_equal(np.array(a)[1:], np.array(b)[1:])
    with pytest.raises(ValueError):
        env2.call("load_checkpoint", [("nobody", ck[0][1])])
