"""Setting and reading an env's physics state: `call("set_state" | "set_env_state" | "get_env_state" | "_get_obs")` of the
vector env and the bare single env's `set_state` / `set_env_state` / `get_env_state` / `_get_obs`.  The REAL host code runs
on the float64 oracle (tests/oracle_state_engine.py, whose set_physics / get_physics / observe do what k_set_physics /
k_get_physics / k_observe do: no forward pass on set, qvel through float32, kinematics before the observation) against the
reference's own stack, step by step.  The reference side is replayed from tests/golden/refstack_<test>.pkl.gz
(tests/refstack_replay.py); with METAWORLD_REFERENCE=<Meta-World checkout> it runs live and rewrites those files."""
import numpy as np
import pytest

from oracle_state_engine import oracle_vec_env as _ours
from refstack_replay import RefSession

KEYS = ("success", "near_object", "grasp_success", "grasp_reward", "in_place_reward", "obj_to_target", "unscaled_reward")
ATOL = 2e-6


@pytest.fixture
def ref(request):
    s = RefSession(request.node.name.replace("[", "_").rstrip("]"))
    yield s
    s.close()


@pytest.fixture
def gym(ref):
    return ref.module("gymnasium")


@pytest.fixture
def metaworld(ref, gym):
    return ref.module("metaworld")


def _same_states(s1, s2):
    """get_env_state tuples: qpos exactly as float64 physics leaves it (to rounding), qvel through the record's float32."""
    assert len(s1) == len(s2)
    for (q1, v1), (q2, v2) in zip(s1, s2):
        assert q1.shape == q2.shape and v1.shape == v2.shape and q2.dtype == v2.dtype == np.float64
        assert np.abs(q1 - q2).max() < 1e-7 and np.abs(v1 - v2).max() < 1e-5


def _same_obs(o1, o2):
    assert len(o1) == len(o2)
    for a, b in zip(o1, o2):
        assert a.shape == b.shape == (39,) and b.dtype == np.float64 and np.abs(a - b).max() < ATOL


def _step_both(ref, ours, a, t):
    r1, r2 = ref.step(a), ours.step(a)
    assert r1[0].dtype == r2[0].dtype and np.abs(r1[0] - r2[0]).max() < ATOL, t
    assert np.abs(r1[1] - r2[1]).max() < 1e-5, t
    assert np.array_equal(r1[2], r2[2]) and np.array_equal(r1[3], r2[3]), t
    f1, f2 = r1[4], r2[4]
    assert set(f1) == set(f2), (t, sorted(f1), sorted(f2))
    for k in (KEYS if "success" in f1 else ()):
        assert np.abs(np.asarray(f1[k], dtype=np.float64) - f2[k]).max() < 1e-5 and np.array_equal(f1["_" + k], f2["_" + k]), (t, k)
    done = r1[2] | r1[3]
    if done.any():
        for e in np.nonzero(done)[0]:
            assert np.abs(f1["final_obs"][e] - f2["final_obs"][e]).max() < ATOL, t
        for k in KEYS:
            assert np.abs(np.asarray(f1["final_info"][k], dtype=np.float64) - f2["final_info"][k]).max() < 1e-5, (t, k)
        assert np.allclose(f1["final_info"]["episode"]["r"], f2["final_info"]["episode"]["r"], atol=1e-3)
    return done


def test_mt10_one_hot_set_state_and_get_obs_match_reference_stack(gym):
    """`call` sends the same arguments to every sub-env.  reach / push / pick-place share nq = 16, nv = 15; door-open (env
    3) has 10 / 10, so push's state is set on envs 0-2 and then fails with MujocoEnv's AssertionError, in both stacks;
    a drawer-close or button-press-topdown state fails at env 0 and sets nothing.  `_get_obs` returns the base env's rows and commits the frame stack,
    and the steps after it (across a truncation) agree."""
    kw = dict(seed=17, use_one_hot=True, max_episode_steps=7, num_goals=3)
    ref = gym.make_vec("Meta-World/MT10", vector_strategy="sync", **kw)
    ours = _ours("mt", "MT10", **kw)
    o1, _ = ref.reset(); o2, _ = ours.reset()
    assert np.abs(o1 - o2).max() < ATOL
    rng = np.random.default_rng(3)
    n_done = 0
    for t in range(12):
        if t in (3, 9):
            s1 = ref.call("get_env_state"); s2 = ours.call("get_env_state")
            _same_states(s1, s2)
            qpos, qvel = s1[1] if t == 3 else s1[5]        # push's state, then drawer-close's
            with pytest.raises(AssertionError):
                ref.call("set_state", qpos, qvel)
            with pytest.raises(AssertionError):
                ours.call("set_state", qpos, qvel)
            s1b = ref.call("get_env_state"); s2b = ours.call("get_env_state")
            _same_states(s1b, s2b)
            changed = [not np.array_equal(a[0], b[0]) for a, b in zip(s1, s1b)]
            assert changed == ([True, False, True] + [False] * 7 if t == 3 else [False] * 10)   # env 1 had this state already
            _same_obs(ref.call("_get_obs"), ours.call("_get_obs"))
        if t == 5:
            st = ref.call("get_env_state")[6]              # button-press-topdown: nq 10 like env 3, not like env 0
            with pytest.raises(AssertionError):
                ref.call("set_env_state", st)
            with pytest.raises(AssertionError):
                ours.call("set_env_state", st)
        a = rng.uniform(-1, 1, size=(10, 4)).astype(np.float32)
        n_done += int(_step_both(ref, ours, a, t).sum())
    assert n_done == 10                                    # every env truncated once, at t = 6
    _same_states(ref.call("get_env_state"), ours.call("get_env_state"))


def test_mt1_set_state_from_another_env_matches_reference(metaworld):
    """MT1 (one task, the wrapped env of make_mt_envs): a state recorded mid-episode is set again later, with
    `set_state` and with `set_env_state`, followed by `_get_obs` or directly by a step, and steps that cross the
    truncation."""
    kw = dict(seed=8, max_episode_steps=9)
    metaworld._N_GOALS = 4
    renv = metaworld.make_mt_envs("pick-place-v3", **kw)
    ours = _ours("mt", "pick-place-v3", num_goals=4, **kw)
    o1, _ = renv.reset(); o2, _ = ours.reset()
    assert np.abs(o1 - o2[0]).max() < ATOL

    def call(name, *args):
        return (renv.get_wrapper_attr(name)(*args),), ours.call(name, *args)

    rng = np.random.default_rng(11)
    saved = None
    for t in range(14):
        if t == 2:
            saved = call("get_env_state")[0][0]
        if t in (5, 7, 11):
            r, o = call("set_state", *saved) if t < 10 else call("set_env_state", saved)
            assert r == o == (None,)
            _same_states(*call("get_env_state"))
            if t != 7:             # at t = 7 the step follows the set directly (the reference's set_state ran mj_forward)
                _same_obs(*call("_get_obs"))
        a = rng.uniform(-1, 1, 4).astype(np.float32)
        a[3] = 1.0 if t % 5 > 2 else a[3]
        x1 = renv.step(a); x2 = ours.step(a[None])
        assert bool(x1[3]) == bool(x2[3][0]), t
        last = x2[4]["final_obs"][0] if x1[3] else x2[0][0]
        assert np.abs(x1[0] - last).max() < ATOL and abs(x1[1] - x2[1][0]) < 1e-5, t
        assert all(abs(float(x1[4][k]) - float((x2[4]["final_info"] if x1[3] else x2[4])[k][0])) < 1e-5 for k in KEYS), t
        if x1[3]:
            o1, _ = renv.reset()
            assert np.abs(o1 - x2[0][0]).max() < ATOL          # our SAME_STEP autoreset already restarted the episode
    _same_states(*call("get_env_state"))


def test_bare_single_env_set_state_matches_reference_class(metaworld):
    """`mt1.train_classes[name]()`: MujocoEnv.set_state's shape assertion, the set_env_state / get_env_state round trip,
    `_get_obs` of the set state (frame stack committed) and the steps after it."""
    from metaworld_b200 import benchmarks as B
    from metaworld_b200.single_env import SawyerXYZEnvB200
    from oracle_state_engine import OracleStateEngine
    metaworld._N_GOALS = 3
    name = "door-open-v3"
    rb = metaworld.MT1(name, seed=2)
    ob = B.MT1(name, seed=2, n_goals=3)
    renv = rb.train_classes[name]()
    oenv = SawyerXYZEnvB200(name, engine=OracleStateEngine([name]))
    renv.set_task(rb.train_tasks[1]); oenv.set_task(ob.train_tasks[1])
    o1, _ = renv.reset(); o2, _ = oenv.reset()
    assert np.abs(o1 - o2).max() < ATOL
    for q, v in ((np.zeros(16), np.zeros(10)), (np.zeros(10), np.zeros(9)), (np.zeros((1, 10)), np.zeros(10))):
        with pytest.raises(AssertionError):
            renv.set_state(q, v)
        with pytest.raises(AssertionError):
            oenv.set_state(q, v)
    rng = np.random.default_rng(4)
    acts = rng.uniform(-1, 1, size=(12, 4)).astype(np.float32)
    saved = None
    for t in range(12):
        if t == 3:
            saved = renv.get_env_state()
            _same_states([saved], [oenv.get_env_state()])
        if t == 8:
            renv.set_env_state(saved); oenv.set_env_state(saved)
            _same_states([renv.get_env_state()], [oenv.get_env_state()])
            _same_states([saved], [oenv.get_env_state()])
            _same_obs([renv._get_obs()], [oenv._get_obs()])
        x1 = renv.step(acts[t]); x2 = oenv.step(acts[t])
        assert np.abs(x1[0] - x2[0]).max() < ATOL and abs(x1[1] - x2[1]) < 1e-5, t
        assert all(abs(float(x1[4][k]) - x2[4][k]) < 1e-5 for k in KEYS), t


def test_vector_set_state_checks_its_inputs():
    """The numpy `set_state` rejects wrong shapes, non-finite values in the columns an env uses and bad masks before
    anything is written; padding columns and unmasked rows are not inspected."""
    v = _ours("mt", "MT10", seed=1, num_goals=2, use_one_hot=True)
    with pytest.raises(RuntimeError):
        v.set_state(np.zeros((10, 18)), np.zeros((10, 17)))          # before reset
    v.reset()
    before = v.call("get_env_state")
    qpos, qvel = (x.numpy() for x in v.get_state_torch())
    assert qpos.shape == (10, 18) and qvel.shape == (10, 17) and not qpos[3, 10:].any() and not qvel[0, 15:].any()
    for q, w in ((qpos[:, :16], qvel), (qpos, qvel[:9]), (qpos[None], qvel)):
        with pytest.raises(ValueError):
            v.set_state(q, w)
    bad = qpos.copy(); bad[3, 9] = np.nan                             # door-open uses qpos[:10]
    with pytest.raises(ValueError):
        v.set_state(bad, qvel)
    with pytest.raises(ValueError):
        v.set_state(qpos, qvel, env_mask=np.ones(10, dtype=np.int64))
    _same_states(before, v.call("get_env_state"))
    bad = qpos.copy(); bad[3, 12] = np.nan; bad[4, 0] = np.inf       # padding of env 3, a row outside the mask
    mask = np.arange(10) != 4
    v.set_state(bad, qvel, env_mask=mask)
    _same_states(before, v.call("get_env_state"))
    # a masked write lands in the masked rows only; observe fills the one-hot columns of the rows it writes
    q2 = qpos.copy(); q2[:, :3] += 0.01
    v.set_state(q2, qvel, env_mask=np.arange(10) == 2)
    after = v.call("get_env_state")
    assert [not np.array_equal(a[0], b[0]) for a, b in zip(before, after)] == [e == 2 for e in range(10)]
    o = v.observe(np.arange(10) == 2)
    assert o.shape == (10, 49) and o.dtype == np.float64 and o[2, 39 + 2] == 1 and np.abs(o[2, :3] - o[2, 18:21]).max() > 0
    assert not o[5, :39].any() and o[5, 39 + 5] == 1
