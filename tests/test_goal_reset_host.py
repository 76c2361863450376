"""CPU suite: episodes at new goals (unfrozen rand_vec).  The C entry points' argument checks in both libraries; the bare
env's `_freeze_rand_vec = False` / `seeded_rand_vec` resets against the reference's own class; and the REAL host code of
`MetaWorldVecEnv.reset_goals` on the float64 oracle stand-in (tests/oracle_engine.py).  The reference side is replayed
from tests/golden/refstack_<test>.pkl.gz (tests/refstack_replay.py); with METAWORLD_REFERENCE=<Meta-World checkout> it
runs live and rewrites those files.  The device side is tests/test_gpu_goal_reset.py."""
import os

import numpy as np
import pytest
import torch

from oracle_engine import OracleEngine, oracle_vec_env
from refstack_replay import gym, metaworld, ref  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_goal_entry_points_reject_a_null_engine(built):
    from metaworld_b200 import engine
    buf = np.zeros(1 << 16, dtype=np.uint8)
    p = buf.ctypes.data
    calls = [("mw_build_goal_rows", (None, p, p, p, p, p, None)), ("mw_build_goal_rows", (None, None, None, None, None, None, None)),
             ("mw_reset_rows", (None, p, p, p, 39, None)), ("mw_reset_rows", (None, None, None, None, 0, None))]
    for so in ("libmwb200.so", "libmwb200_f64.so"):
        lib = engine._load(os.path.join(ROOT, "metaworld_b200", so))
        for name, args in calls:
            assert getattr(lib, name)(*args) == -3, (so, name, args)
            assert lib.mw_last_error().decode() == f"{name}: mw_set_envs not called", (so, name, args)


# reach / pick-place / sweep-into: rejection loops (sweep-into's against its constant goal); drawer-close: reset_model
# moves a static body, and the reset observation shows where the first pass put it
@pytest.mark.parametrize("mode", ["global", "seeded"])
@pytest.mark.parametrize("name", ["reach-v3", "pick-place-v3", "sweep-into-v3", "drawer-close-v3"])
def test_bare_env_unfrozen_resets_match_reference_class(metaworld, name, mode):
    """`mt1.train_classes[name]()` with `_freeze_rand_vec = False`: every reset draws two goals, from the global legacy
    stream ("global", the two sides' streams kept apart by saving and restoring np.random's state) or, with
    `seeded_rand_vec` after `seed(s)`, from the env's own generator.  Over 10 consecutive resets `_last_rand_vec` agrees
    to 1e-12 and the reset observation with the reference's rounded to the engine's float32."""
    from metaworld_b200 import benchmarks as B
    from metaworld_b200.single_env import SawyerXYZEnvB200
    metaworld._N_GOALS = 3
    rb = metaworld.MT1(name, seed=3)
    ob = B.MT1(name, seed=3, n_goals=3)
    renv = rb.train_classes[name]()
    oenv = SawyerXYZEnvB200(name, engine=OracleEngine([name]))
    renv.set_task(rb.train_tasks[0]); oenv.set_task(ob.train_tasks[0])
    renv._freeze_rand_vec = False; oenv._freeze_rand_vec = False
    if mode == "seeded":
        renv.seed(7); oenv.seed(7)
        renv.seeded_rand_vec = True; oenv.seeded_rand_vec = True
    saved = np.random.get_state()
    np.random.seed(11)
    streams = [np.random.get_state(), np.random.get_state()]
    goals = []
    try:
        for k in range(10):
            np.random.set_state(streams[0])
            o1, _ = renv.reset()
            streams[0] = np.random.get_state()
            np.random.set_state(streams[1])
            o2, _ = oenv.reset()
            streams[1] = np.random.get_state()
            r1, r2 = np.asarray(renv._last_rand_vec), oenv._last_rand_vec
            assert r1.shape == r2.shape and np.abs(r1 - r2).max() <= 1e-12, k
            assert o2.shape == (39,) and np.abs(np.asarray(o1).astype(np.float32).astype(np.float64) - o2).max() <= 1e-12, k
            goals.append(r2)
    finally:
        np.random.set_state(saved)
    assert len({g.tobytes() for g in goals}) == 10
    assert oenv.engine.snaps == []      # no reset built a snapshot


def _same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)) or isinstance(a, np.ndarray) and a.dtype == object:
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if a is None or b is None:
        return a is b
    return np.array_equal(a, b)


def test_reset_goals_checks_inputs_and_equals_a_masked_reset_from_snapshots():
    """MT10 x 2 replicas on the oracle with observation normalisation.  `reset_goals` checks its inputs before anything
    changes.  It is, by definition, `engine.reset_masked` from snapshots built for the same goals (twin `u`): same
    observations, wrapper rows and next steps.  It zeroes the episode lengths and ended marks of the masked envs only,
    `get_attr("_last_rand_vec")` reports the new goals, no task-selection draw is consumed (twin `w`, which never calls
    it, holds the same pending draws and RNG states) and the next masked reset draws what `w`'s does."""
    N = 20
    kw = dict(seed=5, num_goals=3, num_envs=N, max_episode_steps=9, normalize_observations=True)
    v, u, w = (oracle_vec_env("mt", "MT10", **kw) for _ in range(3))
    rng = np.random.default_rng(1)
    acts = rng.uniform(-1, 1, size=(8, N, 4)).astype(np.float32)
    mask = np.arange(N) % 2 == 0
    rows = np.nonzero(mask)[0]
    rv, rv1 = v.sample_goals(np.random.default_rng(0), mask)
    with pytest.raises(RuntimeError):
        v.reset_goals(rv, mask, rv1)
    for x in (v, u, w):
        x.reset()
        for a in acts[:3]:
            x.step(a)
    before, ep = v.engine.get_state(), v._ep_len.copy()
    nan = rv.copy(); nan[0, 0] = np.nan
    for args in ((rv[:, :3], mask), (rv.astype(np.float32), mask), (nan, mask), (rv, mask.astype(np.int64)),
                 (rv, mask[:-1]), (rv, mask, nan), (rv, mask, rv1[:1])):
        with pytest.raises(ValueError):
            v.reset_goals(*args)
    assert v.engine.get_state().tobytes() == before.tobytes() and np.array_equal(v._ep_len, ep)
    pending = [(s.pending, s.np_random.bit_generator.state) for s in w.sub]
    obs = v.reset_goals(rv, mask, rv1)
    # the definition, on twin u
    ids = np.zeros(N, dtype=np.int32)
    ids[rows] = u.engine.build_snapshots(u._env_model[rows], rv[rows], u._partial[rows], rand_vec_pass1=rv1[rows])
    d_mask = torch.from_numpy(mask)
    last = u._returned_obs.device()
    u.engine.reset_masked(d_mask, u.d_obs, torch.from_numpy(ids))
    want = u._returned_obs.host().copy()
    want[rows] = u._restarted(d_mask, last).numpy()[rows]
    u._returned_obs.set(host=want)
    assert obs.dtype == want.dtype and np.array_equal(obs, want)
    assert np.array_equal(v._ep_len, np.where(mask, 0, 3)) and not v._autoreset_envs.host().any()
    assert np.array_equal(v.engine.get_state()["snapshot"][rows], -np.ones(len(rows)))
    n = [len(x) for x in w.get_attr("_last_rand_vec")]
    got, old = v.get_attr("_last_rand_vec"), w.get_attr("_last_rand_vec")
    for e in range(N):
        assert np.array_equal(got[e], rv[e, :n[e]] if mask[e] else old[e]), e
    assert v.get_attr("_partially_observable") == w.get_attr("_partially_observable")
    pv, pu, pw = v.post.save_rows(), u.post.save_rows(), w.post.save_rows()
    assert pv.keys() == pu.keys() and all(np.array_equal(np.asarray(pv[k]), np.asarray(pu[k])) for k in pv)
    assert all(np.array_equal(np.asarray(pv[k])[~mask], np.asarray(pw[k])[~mask]) for k in pv)
    assert [(s.pending, s.np_random.bit_generator.state) for s in v.sub] == pending
    # the next steps: the same as the twin's (no episode ends yet: 5 + 0 and 5 + 3 < 9)
    for a in acts[3:8]:
        assert _same(v.step(a), u.step(a))
        w.step(a)
    assert [(s.pending, s.np_random.bit_generator.state) for s in v.sub] == [(s.pending, s.np_random.bit_generator.state) for s in w.sub]
    # the next masked reset draws what it would have drawn without the goal reset
    ov, _ = v.reset(options={"reset_mask": mask})
    ow, _ = w.reset(options={"reset_mask": mask})
    ou, _ = u.reset(options={"reset_mask": mask})
    assert all(np.array_equal(a, b) for a, b in zip(v.get_attr("_last_rand_vec"), w.get_attr("_last_rand_vec")))
    assert np.array_equal(v._d_raw[rows, :39], w._d_raw[rows, :39])
    assert np.array_equal(ov, ou)
