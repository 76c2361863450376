"""GPU suite (-m gpu): episodes at new goals on the device (k_goal_rows, k_reset_rows) and what is built on them: the goal
rows equal the snapshots of the same goals byte for byte, `reset_goals_torch` equals a masked reset from snapshots built
for its goals, never synchronises, keeps the running goal through saves, loads and checkpoints and refuses non-finite
goals; the bare env's unfrozen resets equal its frozen path for the same vectors and never grow the snapshot table."""
import numpy as np
import pytest

from rig import acts, reset_ended, steady_mt50
from rig import torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu


def _without_snapshot(rec):
    """uint8 rows of 512-byte state records (or 768-byte snapshot records) with the snapshot field zeroed."""
    from metaworld_b200.engine import ENVSTATE_DTYPE
    off = ENVSTATE_DTYPE.fields["snapshot"][1]
    r = np.array(rec.view(np.uint8) if rec.dtype.names else rec, dtype=np.uint8, copy=True).reshape(len(rec), -1)
    r[:, off:off + 4] = 0
    return r


@pytest.mark.parametrize("f32", [False, True])
def test_goal_rows_equal_snapshots(torch_cuda, monkeypatch, f32):
    """All 50 tasks x 3 goals (the third with a pass-1 vector of its own), observability alternating: the rows of
    mw_build_goal_rows equal the records mw_build_snapshots makes in the same library, byte for byte except the snapshot
    field (-1 in a row), in precise mode (float64 library) and with MW_B200_SNAPSHOT_F32=1.  Also the entry points' state
    and argument errors on a live engine."""
    torch = torch_cuda
    from metaworld_b200 import engine as E
    from metaworld_b200.benchmarks import draw_rand_vec
    from metaworld_b200.tasks import TASKS
    if f32:
        monkeypatch.setenv("MW_B200_SNAPSHOT_F32", "1")
    names = sorted(TASKS)
    assert len(names) == 50
    eng = E.Engine(names)
    dev = eng.device
    p = torch.zeros(1 << 16, dtype=torch.uint8, device=dev).data_ptr()
    assert E.lib().mw_build_goal_rows(eng.h, p, p, None, p, p, None) == -3          # no env table yet
    assert E.lib().mw_reset_rows(eng.h, p, p, p, 39, None) == -3
    n = 3 * len(names)
    slot = np.repeat(np.arange(len(names)), 3).astype(np.int32)
    eng.set_envs(slot)
    assert E.lib().mw_build_goal_rows(eng.h, None, p, None, p, p, None) == -2
    assert E.lib().mw_reset_rows(eng.h, p, p, p, 38, None) == -2
    rs = np.random.RandomState(9)
    rv, rv1 = np.zeros((n, 6)), np.zeros((n, 6))
    for i, nm in enumerate(names):
        for k in range(3):
            a, b = draw_rand_vec(TASKS[nm], rs), draw_rand_vec(TASKS[nm], rs)
            e = 3 * i + k
            rv[e, :b.size] = b
            rv1[e, :a.size] = a if k == 2 else b
    po = (np.arange(n) % 2).astype(np.uint8)
    ids = eng.build_snapshots(slot, rv, po, rand_vec_pass1=rv1)
    snaps = eng.get_snapshots(int(ids[0]), n)
    rows = torch.full((n, 768), 0xAB, dtype=torch.uint8, device=dev)
    mask = torch.ones(n, dtype=torch.bool, device=dev)
    d = lambda x: torch.from_numpy(x).to(dev)
    eng.build_goal_rows(mask, d(rv), d(rv1), d(po), rows)
    used = 512 + 39 * 4                      # the state record and the observation (the rest of a record is padding)
    got = rows.cpu().numpy()[:, :used]
    want = snaps.view(np.uint8).reshape(n, 768)[:, :used]
    bad = [names[e // 3] for e in range(n) if not np.array_equal(_without_snapshot(got[e:e + 1]), _without_snapshot(want[e:e + 1]))]
    assert not bad, bad
    assert np.all(rows.cpu().numpy().view(E.SNAPSHOT_DTYPE)["st"]["snapshot"].ravel() == -1)
    eng.close()


@pytest.mark.parametrize("mode", ["SameStep", "NextStep", "Disabled"])
def test_reset_goals_torch_equals_a_masked_reset_from_snapshots(torch_cuda, mode):
    """MT50 @ 4096 in steady state, half the envs masked, goals from `sample_goals`: `reset_goals_torch` against a twin
    that builds snapshots for the same goals and restarts from them with `engine.reset_masked`.  Observations, records
    and the outputs of the next 200 steps (DISABLED: the ended envs restart with reset_torch) are bitwise equal, except
    the snapshot field of the rows still on their goal (-1); the unmasked envs' records, hints and observation rows are
    untouched, and the snapshot table does not grow."""
    torch = torch_cuda
    a, b = steady_mt50(torch, mode), steady_mt50(torch, mode)
    N, dev = a.num_envs, a.device
    mask_np = np.arange(N) % 2 == 0
    rows = np.nonzero(mask_np)[0]
    mask = torch.from_numpy(mask_np).to(dev)
    rv, rv1 = a.sample_goals(np.random.default_rng(0), mask_np)
    before = a.save_states()
    obs_before = a._returned_obs.device().clone()
    nsnap = a.engine.get_snapshots(0).shape[0]
    obs_a = a.reset_goals_torch(torch.from_numpy(rv).to(dev), mask, torch.from_numpy(rv1).to(dev)).clone()
    ids = np.zeros(N, dtype=np.int32)
    ids[rows] = b.engine.build_snapshots(b._env_model[rows], rv[rows], b._partial[rows], rand_vec_pass1=rv1[rows])
    last = b._returned_obs.device()
    b.engine.reset_masked(mask, b.d_obs, torch.from_numpy(ids).to(dev))
    obs_b = b._restarted(mask, last).clone()
    assert torch.equal(obs_a, obs_b)
    assert torch.equal(obs_a[~mask], obs_before[~mask])
    sa, sb = a.engine.get_state(), b.engine.get_state()
    assert np.all(sa["snapshot"][rows] == -1)
    assert _without_snapshot(sa).tobytes() == _without_snapshot(sb).tobytes()
    after = a.save_states()
    keep = ~mask
    assert torch.equal(after.records[keep], before.records[keep]) and torch.equal(after.hints[keep], before.hints[keep])
    got = a.get_attr("_last_rand_vec")
    assert all(np.array_equal(got[e], rv[e, :len(got[e])]) for e in rows[:64])
    rng = np.random.default_rng(5)
    for t in range(200):
        act = acts(torch, rng, N, dev)
        oa, ob = a.step_torch(act), b.step_torch(act)
        for x, y in zip(oa, ob):
            assert torch.equal(x, y), (mode, t)
        ra, rb = reset_ended(a, oa), reset_ended(b, ob)
        assert (ra is None and rb is None) or torch.equal(ra, rb), (mode, t)
    sa, sb = a.engine.get_state(), b.engine.get_state()
    still = sa["snapshot"] == -1
    assert still.any() and not still.all()
    assert np.array_equal(sa["snapshot"][~still], sb["snapshot"][~still])
    assert _without_snapshot(sa).tobytes() == _without_snapshot(sb).tobytes()
    assert a.engine.get_snapshots(0).shape[0] == nsnap
    assert not a.engine.faults().any()
    a.close(); b.close()


def test_reset_goals_does_not_synchronise(torch_cuda):
    torch = torch_cuda
    from metaworld_b200.vector_env import make_mt_envs
    env = make_mt_envs("MT10", seed=1, num_envs=200)
    env.reset_torch()
    dev = env.device
    rng = np.random.default_rng(2)
    env.step_torch(acts(torch, rng, 200, dev))
    rv, rv1 = (torch.from_numpy(x).to(dev) for x in env.sample_goals(np.random.default_rng(3)))
    mask = torch.from_numpy(np.arange(200) % 3 == 0).to(dev)
    env.reset_goals_torch(rv, mask, rv1)                 # first use: allocates the buffers, builds the float64 env table
    act = acts(torch, rng, 200, dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        env.reset_goals_torch(rv, ~mask)
        env.step_torch(act)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert not env.engine.faults().any()
    env.close()


def test_fresh_goal_loop(torch_cuda):
    """DISABLED autoreset, 600 steps (horizon 150): the ended envs restart with `reset_goals_torch` at the next goal of
    their own pool (drawn with `sample_goals` up front), chosen on the device.  Every episode starts at its own goal (the
    running goal and `_last_rand_vec` at the end are the pool entry of each env's episode count), with no fault and no
    synchronisation."""
    torch = torch_cuda
    from metaworld_b200.vector_env import make_mt_envs
    N, K = 500, 6
    env = make_mt_envs("MT10", seed=7, num_envs=N, max_episode_steps=150, autoreset_mode="Disabled")
    dev = env.device
    g = np.random.default_rng(11)
    pool = [env.sample_goals(g) for _ in range(K)]
    P = torch.from_numpy(np.stack([p[0] for p in pool])).to(dev)
    P1 = torch.from_numpy(np.stack([p[1] for p in pool])).to(dev)
    env.reset_torch()
    count = torch.zeros(N, dtype=torch.long, device=dev)
    ar = torch.arange(N, device=dev)
    env.reset_goals_torch(P[0], None, P1[0])
    count += 1
    rng = np.random.default_rng(4)
    A = [acts(torch, rng, N, dev) for _ in range(600)]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for t in range(600):
            out = env.step_torch(A[t])
            ended = torch.logical_or(out[2], out[3]).bool()
            k = count.clamp(max=K - 1)
            env.reset_goals_torch(P[k, ar].contiguous(), ended, P1[k, ar].contiguous())
            count += ended
    finally:
        torch.cuda.set_sync_debug_mode("default")
    c = count.cpu().numpy()
    assert c.min() >= 4 and c.max() <= K
    last = env.get_attr("_last_rand_vec")
    pn = np.stack([p[0] for p in pool])
    assert all(np.array_equal(last[e], pn[c[e] - 1, e, :len(last[e])]) for e in range(N))
    assert np.all(env.engine.get_state()["snapshot"] == -1)
    assert not env.engine.faults().any()
    env.close()


def test_goal_state_survives_save_load_and_checkpoint(torch_cuda):
    """NEXT_STEP, MT10 x 10: envs on ad hoc goals are saved and loaded back (load_states_torch), and checkpointed and
    loaded into a new env: both continue bitwise, through autoresets, and report the same `_last_rand_vec`."""
    torch = torch_cuda
    from metaworld_b200.vector_env import make_mt_envs
    N = 100
    mk = lambda: make_mt_envs("MT10", seed=3, num_envs=N, max_episode_steps=25, autoreset_mode="NextStep")
    env = mk()
    dev = env.device
    env.reset_torch()
    rng = np.random.default_rng(6)
    A = [acts(torch, rng, N, dev) for _ in range(70)]
    for a in A[:5]:
        env.step_torch(a)
    rv, rv1 = env.sample_goals(np.random.default_rng(1), np.arange(N) % 2 == 1)
    mask = torch.from_numpy(np.arange(N) % 2 == 1).to(dev)
    env.reset_goals_torch(torch.from_numpy(rv).to(dev), mask, torch.from_numpy(rv1).to(dev))
    for a in A[5:10]:
        env.step_torch(a)

    def run(x, acts):
        return [[y.clone() for y in x.step_torch(a)] for a in acts], x.engine.get_state()

    states = env.save_states()
    goals = env.get_attr("_last_rand_vec")
    ref, st_ref = run(env, A[10:40])
    env.load_states_torch(states)
    assert all(np.array_equal(x, y) for x, y in zip(env.get_attr("_last_rand_vec"), goals))
    got, st_got = run(env, A[10:40])
    assert sum(int(o[3].sum()) for o in ref) > 0
    for t, (p, q) in enumerate(zip(ref, got)):
        assert all(torch.equal(x, y) for x, y in zip(p, q)), t
    assert st_ref.tobytes() == st_got.tobytes()
    # checkpoint: mid-episode, half the envs still on their ad hoc goal
    env.load_states_torch(states)
    ck = env.get_checkpoint()
    new = mk()
    new.load_checkpoint(ck)
    assert all(np.array_equal(x, y) for x, y in zip(new.get_attr("_last_rand_vec"), goals))
    ref, st_ref = run(env, A[10:40])
    got, st_got = run(new, A[10:40])
    for t, (p, q) in enumerate(zip(ref, got)):
        assert all(torch.equal(x, y) for x, y in zip(p, q)), t
    assert st_ref.tobytes() == st_got.tobytes()
    assert not env.engine.faults().any() and not new.engine.faults().any()
    env.close(); new.close()


def test_non_finite_goal_is_refused(torch_cuda):
    """A non-finite goal leaves its env unchanged and sets fault bit 64, alone in its CTA (no donor: no physics runs) and
    next to finite goals; `raise_on_faults()` raises ValueError."""
    torch = torch_cuda
    from metaworld_b200.vector_env import make_mt_envs
    N = 20
    env = make_mt_envs("MT10", seed=2, num_envs=N)
    dev = env.device
    env.reset_torch()
    rv, rv1 = env.sample_goals(np.random.default_rng(0))
    rv[0, 1] = np.nan
    rv1[3, 0] = np.inf
    before = env.engine.get_state()
    mask = torch.zeros(N, dtype=torch.bool, device=dev)
    mask[0] = True
    d = lambda x: torch.from_numpy(x).to(dev)
    env.reset_goals_torch(d(rv), mask, d(rv1))
    assert env.engine.get_state().tobytes() == before.tobytes()
    f = env.engine.faults()
    assert f[0] == 64 and not f[1:].any()
    env.reset_goals_torch(d(rv), None, d(rv1))
    st = env.engine.get_state()
    assert st[0].tobytes() == before[0].tobytes() and st[3].tobytes() == before[3].tobytes()
    ok = np.ones(N, dtype=bool); ok[[0, 3]] = False
    assert np.all(st["snapshot"][ok] == -1) and np.all(st["snapshot"][~ok] >= 0)
    with pytest.raises(ValueError, match="non-finite goal"):
        env.engine.raise_on_faults()
    with pytest.raises(ValueError):
        env.reset_goals(rv, np.ones(N, dtype=bool), rv1)
    env.close()


@pytest.mark.parametrize("name", ["reach-v3", "drawer-close-v3", "basketball-v3"])
def test_bare_env_unfrozen_reset_equals_frozen_path(torch_cuda, name):
    """Five unfrozen resets (np.random seeded) against a second env on the frozen path given the same two vectors
    (`set_task` + `reset(_pass1=...)`): observations bitwise equal, records equal but for the episode counter and the
    snapshot field.  Twenty unfrozen resets do not grow the snapshot table."""
    from metaworld_b200 import benchmarks as B
    from metaworld_b200.single_env import SawyerXYZEnvB200
    from metaworld_b200.tasks import TASKS
    env, fro = SawyerXYZEnvB200(name), SawyerXYZEnvB200(name)
    env.set_task(B.MT1(name, seed=1, n_goals=2).train_tasks[0])
    env._freeze_rand_vec = False
    saved = np.random.get_state()
    np.random.seed(5)
    try:
        for k in range(5):
            st = np.random.get_state()
            o1, _ = env.reset()
            np.random.set_state(st)
            first = B.draw_rand_vec(TASKS[name], np.random)
            second = B.draw_rand_vec(TASKS[name], np.random)
            assert np.array_equal(second, env._last_rand_vec)
            fro.set_task(B.make_task(name, second, env._partially_observable))
            o2, _ = fro.reset(_pass1=first)
            assert np.array_equal(o1, o2), k
            s1, s2 = env.engine.get_state(), fro.engine.get_state()
            for s in (s1, s2):
                s["episode"] = 0; s["snapshot"] = 0
            assert s1.tobytes() == s2.tobytes(), k
            env.step(np.zeros(4)); fro.step(np.zeros(4))
        n0 = env.engine.get_snapshots(0).shape[0]
        for _ in range(20):
            env.reset()
        assert env.engine.get_snapshots(0).shape[0] == n0 == 0
    finally:
        np.random.set_state(saved)
    env.close(); fro.close()


@pytest.mark.parametrize("name", ["reach-v3", "pick-place-v3"])
def test_seeded_rand_vec_reproduces_unfrozen_goals(torch_cuda, name):
    """The reference's test_seeded_rand_vec, made non-vacuous: two goal-observable envs with the same seed,
    `_freeze_rand_vec = False` and `seeded_rand_vec = True` give bit-identical observations and rewards over 3 episodes x
    500 steps, and their goal changes from episode to episode."""
    from metaworld_b200.single_env import make_goal_env
    seed = 123
    e1, e2 = make_goal_env(name, seed=seed, observable=True), make_goal_env(name, seed=seed, observable=True)
    goals = []
    for e in (e1, e2):
        e._freeze_rand_vec = False
        e.seeded_rand_vec = True
    a = -np.ones(4)
    for ep in range(3):
        (o1, _), (o2, _) = e1.reset(), e2.reset()
        assert np.array_equal(o1, o2) and np.array_equal(e1._last_rand_vec, e2._last_rand_vec)
        goals.append(e1._last_rand_vec.copy())
        for t in range(e1.max_path_length):
            s1, s2 = e1.step(a), e2.step(a)
            assert np.array_equal(s1[0], s2[0]) and s1[1] == s2[1], (ep, t)
            assert not s1[2] and not s2[2]
    assert len({g.tobytes() for g in goals}) == 3
    e1.close(); e2.close()
