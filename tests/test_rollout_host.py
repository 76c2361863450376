"""CPU suite: open-loop rollouts (`MetaWorldVecEnv.rollout_torch` / `rollout`).  The C entry point's argument checks in
both libraries, and the REAL host code of the vector env on a float64 oracle stand-in whose `rollout` mirrors k_rollout:
every candidate row starts from a scratch oracle env that replays the env's episode (as `load_states` does) and steps
its actions with TimeLimit and terminate_on_success; the step that ends the episode is the row's last live step.  The
device side is tests/test_gpu_rollout.py."""
import os

import numpy as np
import pytest
import torch

from oracle import mjphys as P
from oracle.tasks import TASKS as OT
from oracle_engine import OracleEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class RolloutOracle(OracleEngine):
    """`OracleEngine` with `rollout` (k_rollout): nothing of the stand-in's envs or bookkeeping changes."""

    def _scratch(self, e):
        """A new oracle env in env e's current state: its episode start, then the calls since, replayed."""
        keep = (self.envs[e], self.snap[e], self.plen[e], self.ret[e], self.ended[e], self.start[e], self.log[e])
        self.envs[e] = OT[self.names[self.env_model[e]]]()
        self._start(e, int(keep[1]), keep[5])
        env = self.envs[e]
        for op in keep[6]:
            if op[0] == "step":
                env.step(op[1])
            elif op[0] == "set":
                env.data.qpos, env.data.qvel = op[1].copy(), op[2].copy()
            else:
                P.mj_forward(env.model, env.data)
                env._get_obs()
        self.envs[e], self.snap[e], self.plen[e], self.ret[e], self.ended[e], self.start[e], self.log[e] = keep
        return env

    def rollout(self, actions, reward, info, flags, obs, diag, hints):
        from metaworld_b200.engine import INFO_KEYS
        a = actions.numpy()
        K, H = a.shape[:2]
        reward.zero_(); info.zero_(); flags.zero_(); diag.zero_()
        if obs is not None:
            obs.zero_()
        for e in range(self.n_envs):
            for k in range(K):
                env = self._scratch(e)
                plen, ended = int(self.plen[e]), bool(self.ended[e]) and self.mode != "SameStep"
                for h in range(H):
                    if ended:
                        flags[k, h, e] = 4
                        continue
                    o, r, _, _, inf = env.step(a[k, h, e])
                    plen += 1
                    tr = plen >= self.max_steps
                    te = self.tos and inf["success"] == 1.0
                    reward[k, h, e] = float(r)
                    info[k, h, e] = torch.tensor([float(inf[n]) for n in INFO_KEYS], dtype=torch.float32)
                    flags[k, h, e] = int(te) + 2 * int(tr)
                    if obs is not None:
                        obs[k, h, e] = torch.from_numpy(o.astype(np.float32))
                    ended = te or tr


def _env(**kw):
    from metaworld_b200 import benchmarks as B
    from metaworld_b200 import vector_env as V
    return V.make_mt_envs("MT10", engine=RolloutOracle(list(dict.fromkeys(B.MT10))), **kw)


def test_rollout_entry_point_rejects_bad_arguments(built):
    from metaworld_b200 import engine
    buf = np.zeros(1 << 16, dtype=np.uint8)
    p = buf.ctypes.data
    good = [1, 1, p, p, p, p, None, p, p, None]          # k, horizon, actions, reward, info, flags, obs, diag, hints, stream
    bad = []
    for i in (2, 3, 4, 5, 7, 8):                         # every required buffer NULL in turn
        args = list(good); args[i] = None; bad.append(args)
    for i in (0, 1):                                     # k or horizon below 1
        for v in (0, -1):
            args = list(good); args[i] = v; bad.append(args)
    for so in ("libmwb200.so", "libmwb200_f64.so"):
        lib = engine._load(os.path.join(ROOT, "metaworld_b200", so))
        for args in bad:
            assert lib.mw_rollout(None, *args) == -2, (so, args)
            assert lib.mw_last_error().decode() == "mw_rollout: bad arguments", (so, args)
        for obs in (None, p):
            args = list(good); args[6] = obs
            assert lib.mw_rollout(None, *args) == -3, so
            assert lib.mw_last_error().decode() == "mw_rollout: mw_set_envs not called", so


def test_rollout_checks_its_inputs_before_changing_anything():
    N = 10
    v = _env(seed=1, num_envs=N, max_episode_steps=9)
    ok = torch.zeros(2, 3, N, 4)
    with pytest.raises(RuntimeError):
        v.rollout_torch(ok)
    with pytest.raises(RuntimeError):
        v.rollout(ok.numpy())
    v.reset()
    v.step(np.zeros((N, 4), np.float32))
    before, ep_len = v.engine.get_state(), v._ep_len.copy()
    for x in (torch.zeros(2, 3, N, 4, dtype=torch.float64), torch.zeros(2, 3, N + 1, 4), torch.zeros(2, 3, N, 3),
              torch.zeros(0, 3, N, 4), torch.zeros(2, 0, N, 4), torch.zeros(3, N, 4), torch.zeros(2, 3, N, 8)[..., :4],
              torch.zeros(2, 3, N, 4, device="meta"), np.zeros((2, 3, N, 4), np.float32)):
        with pytest.raises(ValueError):
            v.rollout_torch(x)
    for x in (np.zeros((2, 3, N, 4)), np.zeros((2, 3, N, 3), np.float32), np.zeros((0, 3, N, 4), np.float32),
              np.zeros((3, N, 4), np.float32)):
        with pytest.raises(ValueError):
            v.rollout(x)
    assert v.engine.get_state().tobytes() == before.tobytes() and np.array_equal(v._ep_len, ep_len)


def _expected(v, st, actions):
    """Fork-and-step under NEXT_STEP (the terminal step reports the terminal observation and its infos): for each
    candidate k, `load_states` the saved state and `step` its actions; the rows' outputs up to and including the step
    that ends each row's episode, zeros and flag 4 after it."""
    assert v.autoreset_mode == "NextStep"
    K, H, N = actions.shape[:3]
    rew, info, flags, obs = np.zeros((K, H, N), np.float32), np.zeros((K, H, N, 7), np.float32), np.zeros((K, H, N), np.uint8), np.zeros((K, H, N, 39), np.float32)
    from metaworld_b200.engine import INFO_KEYS
    for k in range(K):
        v.load_states(st)
        ended = v._autoreset_envs.host().copy()
        for h in range(H):
            o, r, te, tr, inf = v.step(actions[k, h])
            live = ~ended
            rew[k, h] = np.where(live, r, 0)
            info[k, h] = np.where(live[:, None], np.stack([inf[n] for n in INFO_KEYS], 1), 0)
            flags[k, h] = np.where(live, te + 2 * tr, 4)
            obs[k, h] = np.where(live[:, None], o[:, :39], 0)
            ended = ended | te | tr
    return rew, info, flags, obs


def _check(got, want):
    rew, info, flags, obs = want
    assert np.array_equal(got.reward, rew) and np.array_equal(got.info, info) and np.array_equal(got.obs, obs)
    assert np.array_equal(got.terminated, (flags & 1) != 0) and np.array_equal(got.truncated, (flags & 2) != 0)
    assert np.array_equal(got.ended, (flags & 4) != 0)
    assert not got.faults.any() and not got.contacts_dropped.any()


@pytest.mark.parametrize("tos", [False, True])
def test_rows_end_at_the_time_limit_and_on_success(tos):
    """MT10 with max_episode_steps=9, H = 12 from staggered episode lengths: each row truncates at step 8 - path length
    and is ended after it.  With terminate_on_success the reach envs restart at a goal on their hand's start, so their
    rows terminate on the first step.  Outputs equal fork-and-step of the same env."""
    N, K, H = 10, 2, 12
    v = _env(seed=3, num_envs=N, max_episode_steps=9, terminate_on_success=tos, autoreset_mode="NextStep")
    hand = v.reset()[0][:, :3]
    rng = np.random.default_rng(0)
    for t in range(4):
        v.step(rng.uniform(-1, 1, size=(N, 4)).astype(np.float32))
        if t == 1:
            v.reset(options={"reset_mask": np.arange(N) % 2 == 0})     # episode lengths 2 and 4
    reach = np.array([s.task_name == "reach-v3" for s in v.sub])
    if tos:
        rv = np.zeros((N, 6))
        rv[:, :3] = hand + [0.2, 0.2, 0.0]                               # the object, away from the goal
        rv[:, 3:] = hand                                                 # the goal, where the hand starts
        v.reset_goals(rv, reach)
    plen = v._ep_len.copy()
    actions = rng.uniform(-0.1, 0.1, size=(K, H, N, 4)).astype(np.float32)
    st = v.save_states()
    got = v.rollout(actions, obs=True)
    want = _expected(v, st, actions)
    _check(got, want)
    first_end = np.argmax(got.terminated | got.truncated, axis=1)        # [K, N]
    stop = np.where(reach & tos, 0, 8 - plen)
    assert np.array_equal(first_end, np.broadcast_to(stop, (K, N)))
    assert np.array_equal(got.truncated.any(1), np.broadcast_to(~(reach & tos), (K, N)))
    assert np.array_equal(got.terminated.any(1), np.broadcast_to(reach & tos, (K, N)))
    h = np.arange(H)[None, :, None]
    assert np.array_equal(got.ended, np.broadcast_to(h > stop[None, None, :], got.ended.shape))
    assert not got.reward[got.ended].any() and not got.obs[got.ended].any() and not got.info[got.ended].any()


def test_envs_ended_by_the_last_step_are_ended_from_step_0():
    """NEXT_STEP: the rows of the envs whose episode ended in the last step carry flag 4 from step 0 with zero outputs;
    the others equal fork-and-step."""
    N, K, H = 10, 2, 4
    v = _env(seed=4, num_envs=N, max_episode_steps=3, autoreset_mode="NextStep")
    v.reset()
    v.step(np.zeros((N, 4), np.float32))
    v.reset(options={"reset_mask": np.arange(N) < 5})
    for _ in range(2):
        v.step(np.zeros((N, 4), np.float32))
    ended = v._autoreset_envs.host().copy()
    assert ended.any() and not ended.all()
    actions = np.random.default_rng(1).uniform(-1, 1, size=(K, H, N, 4)).astype(np.float32)
    st = v.save_states()
    got = v.rollout(actions, obs=True)
    assert np.array_equal(got.ended[:, 0], np.broadcast_to(ended, (K, N)))
    assert got.ended[:, :, ended].all() and not got.reward[:, :, ended].any() and not got.obs[:, :, ended].any()
    _check(got, _expected(v, st, actions))


@pytest.mark.parametrize("mode", ["SameStep", "NextStep", "Disabled"])
def test_rollout_leaves_the_env_untouched(mode):
    """With every optional wrapper: after a rollout, the `step` outputs (wrapper statistics included), episode lengths and
    records equal those of a twin that did not roll out."""
    N = 10
    kw = dict(seed=6, num_envs=N, max_episode_steps=5, autoreset_mode=mode, normalize_observations=True,
              reward_normalization_method="gymnasium", recurrent_info_in_obs=True)
    v, w = _env(**kw), _env(**kw)
    rng = np.random.default_rng(2)
    A = rng.uniform(-1, 1, size=(10, N, 4)).astype(np.float32)
    outs = []
    for x in (v, w):
        x.reset(seed=6)
        outs.append([x.step(a) for a in A[:3]])
    v.rollout(rng.uniform(-1, 1, size=(2, 4, N, 4)).astype(np.float32), obs=True)
    for x in (v, w):
        out = []
        for a in A[3:]:
            out.append(x.step(a))
            if mode == "Disabled":
                done = out[-1][2] | out[-1][3]
                if done.any():
                    x.reset(options={"reset_mask": done})
        outs.append(out)
    assert v.engine.get_state().tobytes() == w.engine.get_state().tobytes()
    assert np.array_equal(v._ep_len, w._ep_len)
    for a, b in zip(outs[2], outs[3]):
        assert _same(a, b)


def _same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)) or isinstance(a, np.ndarray) and a.dtype == object:
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if a is None or b is None:
        return a is b
    return np.array_equal(a, b)
