"""CPU suite: saved env states (`MetaWorldVecEnv.save_states` / `load_states`).  The C entry points' argument checks in
both libraries, and the REAL host code of the vector env on the float64 oracle stand-in (tests/oracle_engine.py, whose
save_states / load_states replay a saved row's episode on the target env): the host mirrors, the optional wrappers' rows
and the returned observations follow `src`, and a restored env replays the original run exactly, also from a state
saved on a goal row.  The device side is tests/test_gpu_branch.py."""
import os

import numpy as np
import pytest

from oracle_engine import oracle_vec_env as _ours

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_save_and_load_entry_points_reject_bad_arguments(built):
    from metaworld_b200 import engine
    buf = np.zeros(1 << 16, dtype=np.uint8)
    p = buf.ctypes.data
    calls = [("mw_save_states", (None, p, p, p, p, None)), ("mw_save_states", (None, p, None, p, p, None)),
             ("mw_save_states", (None, None, p, p, None, None)),
             ("mw_load_states", (None, p, p, 1, p, p, p, None)), ("mw_load_states", (None, None, None, 1, None, p, p, None)),
             ("mw_load_states", (None, p, p, -1, p, p, p, None)), ("mw_load_states", (None, p, p, 1, p, p, None, None))]
    for so in ("libmwb200.so", "libmwb200_f64.so"):
        lib = engine._load(os.path.join(ROOT, "metaworld_b200", so))
        for name, args in calls:
            assert getattr(lib, name)(*args) == -2, (so, name, args)
            assert lib.mw_last_error().decode() == f"{name}: bad arguments", (so, name, args)


def _same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)) or isinstance(a, np.ndarray) and a.dtype == object:
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if a is None or b is None:
        return a is b
    return np.array_equal(a, b)


def _run(v, acts):
    return [v.step(a) for a in acts]


def test_load_restores_ended_marks_mirrors_wrapper_rows_and_replays():
    """MT10 x 3 replicas on the oracle, NEXT_STEP, every optional wrapper.  A masked reset staggers the episodes, so at the
    save some envs have just ended and the others are mid-episode.  Loading with `src` permuted among the envs of each
    type gives every env its source's episode length, ended mark, running task, wrapper rows and last observation;
    loading the save back with `src` = identity replays the original steps exactly (observations, rewards, flags,
    infos with the episode statistics, path lengths)."""
    N = 30
    v = _ours("mt", "MT10", seed=5, num_goals=3, num_envs=N, max_episode_steps=9, autoreset_mode="NextStep",
              normalize_observations=True, reward_normalization_method="gymnasium", recurrent_info_in_obs=True)
    with pytest.raises(RuntimeError):
        v.save_states()
    v.reset()
    rng = np.random.default_rng(0)
    acts = rng.uniform(-1, 1, size=(14, N, 4)).astype(np.float32)
    _run(v, acts[:3])
    v.reset(options={"reset_mask": np.arange(N) % 3 == 0})
    last = _run(v, acts[3:9])[-1][0]
    v.call("toggle_sample_tasks_on_reset", False)         # a restart then draws the same task in both runs
    st = v.save_states()
    ep_len, ended = v._ep_len.copy(), v._autoreset_envs.host().copy()
    assert ended.any() and not ended.all() and len(set(ep_len)) > 1
    rv = v.get_attr("_last_rand_vec")
    post = v.post.save_rows()
    orig = _run(v, acts[9:14])
    orig_len = v.get_attr("curr_path_length")
    # permuted within each env type (env e has type e % 10)
    src = np.arange(N).reshape(3, 10)[[1, 2, 0]].reshape(-1)
    obs = v.load_states(st, src=src)
    assert np.array_equal(v._ep_len, ep_len[src]) and np.array_equal(v._autoreset_envs.host(), ended[src])
    assert all(np.array_equal(x, rv[s]) for x, s in zip(v.get_attr("_last_rand_vec"), src))
    rows = v.post.save_rows()
    assert rows.keys() == post.keys() and all(np.array_equal(rows[k], post[k][src]) for k in post)
    assert np.array_equal(obs, last[src])
    # a mask and identity: only the masked rows change
    m = np.arange(N) < 10
    obs = v.load_states(st, env_mask=m)
    assert np.array_equal(obs[:10], last[:10]) and np.array_equal(obs[10:], last[src][10:])
    obs = v.load_states(st)
    assert np.array_equal(obs, last)
    got = _run(v, acts[9:14])
    assert any(x[4].get("_episode", np.zeros(1)).any() for x in orig)      # the window holds episode ends
    for t, (a, b) in enumerate(zip(orig, got)):
        assert _same(a, b), t
    assert v.get_attr("curr_path_length") == orig_len


def test_state_saved_on_a_goal_row_replays():
    """MT10 x 2 replicas on the oracle: every other env restarts at a new goal (`reset_goals`) and is saved two steps
    later, while it runs on its goal row.  Loading the save back with `src` = identity restores the running goals and
    replays the following steps exactly, through the episode ends in the window."""
    N = 20
    v = _ours("mt", "MT10", seed=3, num_goals=2, num_envs=N, max_episode_steps=6)
    v.reset()
    acts = np.random.default_rng(1).uniform(-1, 1, size=(9, N, 4)).astype(np.float32)
    _run(v, acts[:1])
    mask = np.arange(N) % 2 == 0
    rv, rv1 = v.sample_goals(np.random.default_rng(0), mask)
    v.reset_goals(rv, mask, rv1)
    _run(v, acts[1:3])
    v.call("toggle_sample_tasks_on_reset", False)         # a restart then draws the same task in both runs
    st = v.save_states()
    assert np.all(v.engine.get_state()["snapshot"][mask] == -1)
    goals = v.get_attr("_last_rand_vec")
    orig = _run(v, acts[3:])
    assert any(x[3].any() for x in orig)                  # the window holds episode ends
    v.load_states(st, src=np.arange(N))
    assert all(np.array_equal(x, y) for x, y in zip(v.get_attr("_last_rand_vec"), goals))
    got = _run(v, acts[3:])
    for t, (a, b) in enumerate(zip(orig, got)):
        assert _same(a, b), t


def test_load_checks_its_inputs_before_changing_anything():
    v = _ours("mt", "MT10", seed=2, num_goals=2, num_envs=20, max_episode_steps=6)
    w = _ours("mt", "MT10", seed=2, num_goals=2, num_envs=20, max_episode_steps=6)
    v.reset(); w.reset()
    st = v.save_states(np.arange(20) < 15)
    v.step(np.zeros((20, 4), np.float32))
    before = v.engine.get_state()
    for kw in (dict(src=np.roll(np.arange(20), 1)),            # another model
               dict(src=np.full(20, 20)),                        # out of range
               dict(env_mask=np.arange(20) == 17)):              # a row that was not saved
        with pytest.raises(ValueError):
            v.load_states(st, **kw)
    with pytest.raises(ValueError):
        w.load_states(st)                                        # saved by another env
    with pytest.raises(ValueError):
        v.load_states(st, env_mask=np.ones(20, dtype=np.int64))
    assert v.engine.get_state().tobytes() == before.tobytes() and np.array_equal(v._ep_len, np.ones(20))
    e = np.arange(20)
    v.load_states(st, env_mask=(e < 15) | (e == 19), src=np.where(e == 19, 9, e))
    assert np.array_equal(v._ep_len, np.where((e < 15) | (e == 19), 0, 1))
