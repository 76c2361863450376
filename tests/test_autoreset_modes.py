"""gymnasium's NEXT_STEP and DISABLED autoreset modes and `reset(options={"reset_mask": ...})`: the REAL `MetaWorldVecEnv`
host code on the float64 oracle (tests/oracle_engine.py) against the reference's own `gym.make_vec(..., autoreset_mode=...)`
stack, step by step.  The reference side is replayed from tests/golden/refstack_<test>.pkl.gz (tests/refstack_replay.py);
with METAWORLD_REFERENCE=<Meta-World checkout> it runs live and rewrites those files."""
import numpy as np
import pytest

from oracle_engine import oracle_vec_env as _ours
from refstack_replay import RefSession

KEYS = ("success", "near_object", "grasp_success", "grasp_reward", "in_place_reward", "obj_to_target", "unscaled_reward")


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


def _same_obs(o1, o2, atol):
    assert o1.shape == o2.shape and o1.dtype == o2.dtype and np.abs(o1 - o2).max() < atol


def _compare_infos(f1, f2, t):
    assert set(f1) == set(f2), (t, sorted(f1), sorted(f2))
    assert "final_obs" not in f2 and "final_info" not in f2
    for k in (KEYS if "success" in f1 else ()):
        assert np.abs(np.asarray(f1[k], dtype=np.float64) - f2[k]).max() < 1e-5 and np.array_equal(f1["_" + k], f2["_" + k]), (t, k)
    if "episode" in f1:
        e1, e2 = f1["episode"], f2["episode"]
        assert np.array_equal(f1["_episode"], f2["_episode"]) and np.array_equal(e1["_r"], e2["_r"]), t
        assert np.array_equal(e1["l"], e2["l"]) and np.allclose(e1["r"], e2["r"], atol=1e-3), t


def _reset_mask(env, mask):
    opts = {"reset_mask": mask}
    out = env.reset(options=opts)
    opts["reset_mask"] = mask         # gymnasium pops the mask from the caller's dict (and the recording holds that dict)
    return out


def _rollout(ref, ours, mode, steps, seed, atol=2e-6, masks=None):
    """Steps both stacks with the same actions; under DISABLED every finished env is reset with `reset_mask` right away.
    `masks`: {step: bool mask} of extra partial resets before that step.  Returns (episodes ended, restarts seen)."""
    n = ours.num_envs
    rng = np.random.default_rng(seed)
    n_done = n_restart = 0
    prev_done = np.zeros(n, dtype=bool)
    for t in range(steps):
        if masks and t in masks:
            (o1, i1), (o2, i2) = _reset_mask(ref, masks[t]), _reset_mask(ours, masks[t].copy())
            _same_obs(o1, o2, atol)
            assert i1 == i2 == {}
            prev_done &= ~masks[t]
        a = rng.uniform(-1, 1, size=(n, 4)).astype(np.float32)
        a[:, 3] = 1.0 if t % 7 > 3 else a[:, 3]
        r1, r2 = ref.step(a), ours.step(a)
        _same_obs(r1[0], r2[0], atol)
        assert r1[1].dtype == r2[1].dtype and np.abs(r1[1] - r2[1]).max() < 1e-5, t
        assert np.array_equal(r1[2], r2[2]) and np.array_equal(r1[3], r2[3]), t
        _compare_infos(r1[4], r2[4], t)
        if mode == "NextStep" and prev_done.any():       # the restart call: reward 0, no flags, no infos for those envs
            n_restart += int(prev_done.sum())
            assert not r2[1][prev_done].any() and not (r2[2] | r2[3])[prev_done].any()
            assert "success" not in r2[4] or not r2[4]["_success"][prev_done].any()
        done = r1[2] | r1[3]
        n_done += int(done.sum())
        if mode == "Disabled" and done.any():
            (o1, i1), (o2, i2) = _reset_mask(ref, done.copy()), _reset_mask(ours, done.copy())
            _same_obs(o1, o2, atol)
            assert i1 == i2 == {}
            done = np.zeros(n, dtype=bool)
        prev_done = done
        rv1, rv2 = ref.get_attr("_last_rand_vec"), ours.get_attr("_last_rand_vec")
        assert all(np.array_equal(x, y) for x, y in zip(rv1, rv2)), t
    return n_done, n_restart


@pytest.mark.parametrize("mode", ["NextStep", "Disabled"])
def test_mt10_one_hot_autoreset_mode_matches_reference_stack(gym, mode):
    kw = dict(seed=42, use_one_hot=True, max_episode_steps=6, terminate_on_success=True, num_goals=3, autoreset_mode=mode)
    ref = gym.make_vec("Meta-World/MT10", vector_strategy="sync", **kw)
    ours = _ours("mt", "MT10", **kw)
    o1, _ = ref.reset(); o2, _ = ours.reset()
    _same_obs(o1, o2, 2e-6)
    n_done, n_restart = _rollout(ref, ours, mode, 26, seed=1)
    assert n_done >= 30 and (n_restart >= 20 or mode == "Disabled")


@pytest.mark.parametrize("mode", ["NextStep", "Disabled"])
def test_ml10_train_autoreset_mode_matches_reference_stack(gym, metaworld, mode):
    kw = dict(seed=7, meta_batch_size=20, max_episode_steps=5, autoreset_mode=mode)
    metaworld._N_GOALS = 4
    ref = gym.make_vec("Meta-World/ML10-train", vector_strategy="sync", **kw)
    ours = _ours("ml", "ML10", split="train", num_goals=4, **kw)
    ref.call("toggle_sample_tasks_on_reset", True); ours.call("toggle_sample_tasks_on_reset", True)
    o1, _ = ref.reset(); o2, _ = ours.reset()
    _same_obs(o1, o2, 2e-6)
    n_done, _ = _rollout(ref, ours, mode, 17, seed=5)
    assert n_done >= 40


@pytest.mark.parametrize("extra", [dict(reward_normalization_method="gymnasium", normalize_observations=True),
                                   dict(recurrent_info_in_obs=True, normalize_observations=True, reward_normalization_method="exponential"),
                                   dict(recurrent_info_in_obs=True, normalize_reward_in_recurrent_info=False, reward_normalization_method="gymnasium")])
def test_next_step_with_normalisation_and_recurrent_wrappers_matches_reference_stack(gym, extra):
    """The optional wrappers under NEXT_STEP: the terminal step is a plain step, and the restart call is a reset for the
    restarted envs (zero recurrent extension, observation statistics see the reset observation, reward 0 not normalised)."""
    kw = dict(seed=11, use_one_hot=True, max_episode_steps=7, terminate_on_success=True, num_goals=2, autoreset_mode="NextStep", **extra)
    ref = gym.make_vec("Meta-World/MT10", vector_strategy="sync", **kw)
    ours = _ours("mt", "MT10", **kw)
    o1, _ = ref.reset(); o2, _ = ours.reset()
    _same_obs(o1, o2, 3e-4)
    masks = {12: np.arange(10) % 3 == 0}          # and a partial reset of wrapped envs
    n_done, n_restart = _rollout(ref, ours, "NextStep", 25, seed=4, atol=3e-4, masks=masks)
    assert n_done >= 20 and n_restart >= 15


def test_partial_resets_with_reset_mask_match_reference_stack(gym):
    """`reset(options={"reset_mask": m})` mid-episode, under SAME_STEP as well as NEXT_STEP: only the masked envs take a
    task-select draw and restart; the other rows are the envs' latest observations."""
    for mode in ("SameStep", "NextStep"):
        kw = dict(seed=3, use_one_hot=True, max_episode_steps=8, num_goals=4, autoreset_mode=mode)
        ref = gym.make_vec("Meta-World/MT10", vector_strategy="sync", **kw)
        ours = _ours("mt", "MT10", **kw)
        o1, _ = ref.reset(); o2, _ = ours.reset()
        _same_obs(o1, o2, 2e-6)
        masks = {3: np.arange(10) % 2 == 0, 5: np.arange(10) == 7, 11: np.arange(10) >= 4}
        if mode == "SameStep":
            for t in range(14):
                if t in masks:
                    (r1, _), (r2, _) = _reset_mask(ref, masks[t]), _reset_mask(ours, masks[t].copy())
                    _same_obs(r1, r2, 2e-6)
                a = np.random.default_rng(t).uniform(-1, 1, size=(10, 4)).astype(np.float32)
                x1, x2 = ref.step(a), ours.step(a)
                _same_obs(x1[0], x2[0], 2e-6)
                assert np.array_equal(x1[2] | x1[3], x2[2] | x2[3])
                assert all(np.array_equal(x, y) for x, y in zip(ref.get_attr("_last_rand_vec"), ours.get_attr("_last_rand_vec")))
        else:
            _rollout(ref, ours, mode, 14, seed=2, masks=masks)


def test_next_step_checkpoint_between_terminal_step_and_restart(gym):
    """A checkpoint taken right after a terminal step shows the task and task-select RNG state from before the next
    task's draw; each side loads the other's and the restart call draws the same next task."""
    kw = dict(seed=21, use_one_hot=True, max_episode_steps=4, num_goals=3, autoreset_mode="NextStep")
    ref = gym.make_vec("Meta-World/MT10", vector_strategy="sync", **kw)
    ours = _ours("mt", "MT10", **kw)
    o1, _ = ref.reset(); o2, _ = ours.reset()
    _same_obs(o1, o2, 2e-6)
    _rollout(ref, ours, "NextStep", 4, seed=9)        # the 4th step truncates every env
    c1, c2 = ref.call("get_checkpoint"), ours.call("get_checkpoint")
    for (id1, d1), (id2, d2) in zip(c1, c2):
        assert id1 == id2 and d1["rng_state"] == d2["rng_state"] and d1["env_rng_state"]["np_random_state"] == d2["env_rng_state"]["np_random_state"]
        assert d2["mw_b200"]["ep_len"] == 4
    rv_before = ours.get_attr("_last_rand_vec")
    ours.call("load_checkpoint", list(c1))
    ref.call("load_checkpoint", list(c2))
    assert all(np.array_equal(x, y) for x, y in zip(rv_before, ours.get_attr("_last_rand_vec")))
    n_done, n_restart = _rollout(ref, ours, "NextStep", 9, seed=10)
    assert n_restart >= 10 and n_done >= 10


def test_disabled_mode_refuses_to_step_an_ended_env(gym):
    kw = dict(seed=5, max_episode_steps=2, num_goals=2, autoreset_mode="Disabled")
    ref = gym.make_vec("Meta-World/MT10", vector_strategy="sync", **kw)
    ours = _ours("mt", "MT10", **kw)
    ref.reset(); ours.reset()
    a = np.zeros((10, 4), np.float32)
    for _ in range(2):
        x1, x2 = ref.step(a), ours.step(a)
    assert x1[3].all() and x2[3].all()
    with pytest.raises(AssertionError):
        ref.step(a)
    with pytest.raises(AssertionError):
        ours.step(a)
    mask = np.arange(10) < 10
    (o1, _), (o2, _) = _reset_mask(ref, mask), _reset_mask(ours, mask.copy())
    _same_obs(o1, o2, 2e-6)
    x1, x2 = ref.step(a), ours.step(a)
    _same_obs(x1[0], x2[0], 2e-6)


def test_autoreset_mode_spellings_and_forwarding():
    from metaworld_b200 import entry_points
    from metaworld_b200.vector_env import parse_autoreset_mode
    from oracle.refshim.gymnasium.vector import AutoresetMode
    from oracle_engine import OracleEngine
    for m in AutoresetMode:
        assert parse_autoreset_mode(m) == parse_autoreset_mode(m.value) == m.value
    assert parse_autoreset_mode(None) == "SameStep"
    for bad in ("same_step", "NEXT_STEP", 1, "", object()):
        with pytest.raises(ValueError):
            parse_autoreset_mode(bad)
    table = entry_points()
    names = ["reach-v3", "push-v3"]
    v = table["custom-mt-envs"][1](envs_list=names, seed=1, num_goals=2, engine=OracleEngine(names))
    assert v.autoreset_mode == "SameStep" and v.metadata["autoreset_mode"] == "same_step"
    v = table["custom-mt-envs"][1](envs_list=names, seed=1, num_goals=2, autoreset_mode=AutoresetMode.NEXT_STEP, engine=OracleEngine(names))
    assert v.autoreset_mode == "NextStep" and v.metadata["autoreset_mode"] == "next_step"
    assert type(v).metadata["autoreset_mode"] == "same_step"          # per instance
    v = table["MT1"][1](env_name="reach-v3", seed=1, num_goals=2, autoreset_mode="Disabled", engine=OracleEngine(["reach-v3"]))
    assert v.metadata["autoreset_mode"] == "disabled"
    v = table["ML1-train"][1](env_name="reach-v3", seed=1, meta_batch_size=2, num_goals=2, autoreset_mode="Disabled", engine=OracleEngine(["reach-v3"]))
    assert v.autoreset_mode == "Disabled"
    v = table["custom-ml-envs"][1](train_envs=names, test_envs=["door-open-v3"], seed=1, meta_batch_size=2, num_goals=2,
                                   autoreset_mode="NextStep", engine=OracleEngine(names))
    assert v.autoreset_mode == "NextStep"
    with pytest.raises(ValueError):
        table["MT10"][1](seed=1, num_goals=2, autoreset_mode="Sometimes", engine=OracleEngine(["reach-v3"]))
    s = table["MT1"][0](env_name="reach-v3", seed=1, num_goals=2, autoreset_mode="Disabled", engine=OracleEngine(["reach-v3"]))
    assert s.reset()[0].shape == (39,)           # the gym.make form ignores the argument, like the reference
