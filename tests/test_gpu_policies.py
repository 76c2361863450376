"""GPU suite (-m gpu): the scripted expert policies on the device (k_expert, `expert_actions_torch`, metaworld_b200.policies).

  * k_expert equals the host build of the same header (tests/test_policies.py checks that one against the reference's
    policy code) bit for bit;
  * the reference's acceptance test (tests/metaworld/envs/mujoco/sawyer_xyz/test_scripted_policies.py: 50 goals per task,
    closed loop, success >= 80 %) runs closed loop on the device, and so does its `test_evaluation` (MT50, 50 episodes per
    task);
  * `expert_actions_torch()` without an argument reads the base observation the last reset / step left."""
import os

import numpy as np
import pytest

from rig import POLICY_FAILS_ON_REFERENCE_GLUE, _report
from rig import torch_cuda  # noqa: F401
from test_policies import ALL_SOURCES, build_shim, expert_rows, host_actions

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
N_GOALS, MAX_STEPS = 50, 500
# Below the bar on the restated physics itself, measured closed loop on the float64 oracle with the host build of the same
# policies (so not a device parity gap): within `evaluation`'s 300-step episodes soccer's policy solves 36 of MT50's 50
# soccer goals (seed 42) on the oracle; the device scored 0.76 there.  At 500 steps (the acceptance test) it reaches 0.80 on
# both.
BELOW_BAR_AT_300_STEPS = {"soccer-v3": "soccer's policy solves 36/50 of MT50's goals within 300 steps on the float64 oracle too"}


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return build_shim(str(tmp_path_factory.mktemp("devpolicy") / "libdevpolicy.so"))


def _tasks():
    from metaworld_b200.tasks import TASK_IDS
    return sorted(TASK_IDS)


def test_kernel_equals_host_build_bitwise(torch_cuda, shim):
    """Every observation of the trajectory goldens (~1000 per task), two layouts: packed (stride 39) and with 50 one-hot
    columns behind the base observation (stride 89, the one-hot columns set to garbage that must not matter).  Unknown task
    ids give NaN rows."""
    torch = torch_cuda
    from metaworld_b200.engine import expert_actions
    from metaworld_b200.tasks import TASK_IDS
    rows = {t: expert_rows(t, ALL_SOURCES) for t in _tasks()}
    obs = np.concatenate([rows[t] for t in _tasks()])
    ids = np.concatenate([np.full(len(rows[t]), TASK_IDS[t], np.int32) for t in _tasks()])
    ids[:7] = [-1, 50, 1000, -(2 ** 31), 50, -1, 77]
    want = host_actions(shim, ids, obs.astype(np.float64))
    assert np.isnan(want[:7]).all() and np.isfinite(want[7:]).all()
    wide = np.concatenate([obs, np.random.default_rng(0).normal(size=(len(obs), 50)).astype(np.float32)], 1)
    d_ids = torch.from_numpy(ids).cuda()
    for o in (obs, wide):
        d_obs = torch.from_numpy(np.ascontiguousarray(o)).cuda()
        out = torch.full((len(o), 4), 7.0, device="cuda")
        expert_actions(d_ids, d_obs, out)
        got = out.cpu().numpy()
        assert np.isnan(got[:7]).all()
        assert got[7:].tobytes() == want[7:].tobytes()
    # a strided view: the first 39 columns of the wide table
    out = torch.empty(len(obs), 4, device="cuda")
    expert_actions(d_ids, torch.from_numpy(wide).cuda()[:, :45], out)
    assert out.cpu().numpy()[7:].tobytes() == want[7:].tobytes()


def test_policy_objects_match_the_batch(torch_cuda):
    """`ENV_POLICY_MAP[name]().get_action(obs)` on one row equals that row of the batched call; the reference's checks and
    warning come along."""
    from metaworld_b200 import policies
    g = np.load(os.path.join(GOLD, "expert_actions.npz"))
    for t in ("pick-place-v3", "button-press-v3", "handle-pull-v3", "drawer-open-v3"):
        obs = expert_rows(t).astype(np.float64)
        pol = policies.ENV_POLICY_MAP[t]()
        batch = pol.get_actions(obs)
        assert batch.dtype == np.float32 and batch.shape == (len(obs), 4)
        for i in (0, len(obs) // 3, len(obs) - 1):
            a = pol.get_action(obs[i])
            assert a.dtype == np.float32 and a.tobytes() == batch[i].tobytes()
        np.testing.assert_allclose(batch, g[f"{t}/actions"], rtol=1e-6, atol=1e-6)
    pol = policies.SawyerDrawerOpenV3Policy()
    with pytest.raises(AssertionError, match="Observation not fully parsed"):
        pol.get_action(np.zeros(40))
    far = np.zeros(39)
    far[4:7] = [0.0, 0.9, 0.1]
    with pytest.warns(UserWarning, match="Constant"):
        pol.get_action(far)


def _oracle_rate(shim, task, goals):
    """The same goals closed loop on the float64 oracle, driven by the host build of the policies: the success rate."""
    from oracle.tasks import TASKS
    from metaworld_b200.tasks import TASK_IDS
    wins = 0
    for tk in goals:
        env = TASKS[task]()
        env.set_task_vec(tk.unpack()["rand_vec"], False)
        obs, _ = env.reset()
        for _ in range(MAX_STEPS):
            obs, _, _, _, info = env.step(host_actions(shim, [TASK_IDS[task]], obs[None])[0])
            if info["success"]:
                wins += 1
                break
    return wins / len(goals)


@pytest.fixture(scope="module")
def acceptance_rates(torch_cuda):
    """The reference's acceptance test for all 50 tasks in one launch: 50 tasks x the 50 train goals of MT1(task, seed=42)
    = 2500 envs, one fixed goal each, `step_torch(expert_actions_torch())` for up to 500 steps; first success per env."""
    torch = torch_cuda
    from metaworld_b200 import benchmarks as B
    from metaworld_b200.vector_env import MetaWorldVecEnv
    names, tasks = [], []
    for t in _tasks():
        goals = B.MT1(t, seed=42).train_tasks
        assert len(goals) == N_GOALS
        names += [t] * N_GOALS
        tasks += [[g] for g in goals]
    env = MetaWorldVecEnv(names, tasks, seed=42, max_episode_steps=MAX_STEPS)
    env.reset_torch()
    ok = torch.zeros(env.num_envs, dtype=torch.bool, device=env.device)
    for _ in range(MAX_STEPS):
        _, _, term, trunc, info = env.step_torch(env.expert_actions_torch())
        ok |= info[:, 0] == 1.0
        done = (term | trunc) != 0
        ok |= done & (env.d_final_info[:, 0] == 1.0)
    assert not env.engine.faults().any()
    wins = ok.view(len(_tasks()), N_GOALS).sum(1).cpu().numpy()
    rates = [int(w) / N_GOALS for w in wins]
    env.close()
    return dict(zip(_tasks(), rates))


@pytest.mark.parametrize("task", [pytest.param(t, marks=pytest.mark.xfail(reason=POLICY_FAILS_ON_REFERENCE_GLUE[t], strict=False))
                                  if t in POLICY_FAILS_ON_REFERENCE_GLUE else t for t in _tasks()])
def test_scripted_policy_succeeds_closed_loop(acceptance_rates, shim, task):
    g = np.load(os.path.join(GOLD, f"traj_{task}.npz"))
    rate = acceptance_rates[task]
    print(f"POLICY {task}: device closed loop {rate:.2f} (50 goals), reference glue {int(g['s_success'].sum())}/5")
    _report("policy_closed_loop.csv", f"{task},{rate:.2f},{int(g['s_success'].sum())}\n")
    if rate < 0.8 and task not in POLICY_FAILS_ON_REFERENCE_GLUE:
        from metaworld_b200 import benchmarks as B
        oracle = _oracle_rate(shim, task, B.MT1(task, seed=42).train_tasks)
        pytest.fail(f"{task}: device closed loop {rate:.2f} < 0.8; the float64 oracle with the same policy: {oracle:.2f}")
    assert rate >= 0.8


def test_reference_evaluation_with_scripted_agent(torch_cuda):
    """The reference's tests/metaworld/test_evaluation.py: `evaluation()` over MT50 (max 300 steps per episode) with an
    agent that plays the scripted policies, 50 episodes per task."""
    from metaworld_b200 import evaluation as E
    from metaworld_b200 import policies
    from metaworld_b200.vector_env import make_mt_envs
    env = make_mt_envs("MT50", seed=42, max_episode_steps=300)
    names = list(env.get_attr("task_name"))

    class ScriptedAgent:
        def eval_action(self, obs):
            return policies.get_actions(obs, names)

        def reset(self, mask):
            pass

    mean, _, per_task, _ = E.evaluation(ScriptedAgent(), env, num_episodes=50)
    env.close()
    print("EVALUATION", {k: round(v, 2) for k, v in per_task.items()})
    _report("policy_evaluation.csv", "".join(f"{k},{v:.2f}\n" for k, v in per_task.items()))
    assert mean >= 0.8
    excused = set(POLICY_FAILS_ON_REFERENCE_GLUE) | set(BELOW_BAR_AT_300_STEPS)
    low = {k: v for k, v in per_task.items() if v < 0.8 and k not in excused}
    assert not low, low


def test_default_observation_source(torch_cuda):
    """`expert_actions_torch()` equals the call on the base observation the last reset / step wrote, in every case."""
    torch = torch_cuda
    from metaworld_b200.vector_env import make_mt_envs
    rng = np.random.default_rng(3)

    def actions(n):
        return rng.uniform(-1, 1, size=(n, 4)).astype(np.float32)

    # numpy reset / step, one-hot: the explicit observation is what the numpy API returned (first 39 columns)
    env = make_mt_envs("MT10", seed=1, num_envs=20, use_one_hot=True, max_episode_steps=5)
    obs, _ = env.reset()
    assert obs.shape == (20, 49)
    a0 = env.expert_actions()
    assert a0.tobytes() == env.expert_actions(obs).tobytes()
    for _ in range(7):                                         # crosses a truncation + autoreset
        obs, *_ = env.step(actions(20))
        assert env.expert_actions().tobytes() == env.expert_actions(obs).tobytes()
    # masked numpy reset after a numpy step: reset rows and stepped rows together
    m = np.zeros(20, dtype=bool); m[::3] = True
    obs, _ = env.reset(options={"reset_mask": m})
    assert env.expert_actions().tobytes() == env.expert_actions(obs).tobytes()
    # torch calls; a masked reset_torch right after the numpy call
    mt = torch.zeros(20, dtype=torch.bool, device=env.device); mt[1::4] = True
    o = env.reset_torch(mt)
    assert torch.equal(env.expert_actions_torch(), env.expert_actions_torch(o))
    for _ in range(6):
        o, *_ = env.step_torch(torch.from_numpy(actions(20)).to(env.device))
        assert torch.equal(env.expert_actions_torch(), env.expert_actions_torch(o))
    o = env.reset_torch(mt)
    assert torch.equal(env.expert_actions_torch(), env.expert_actions_torch(o))
    o = env.reset_torch()
    assert torch.equal(env.expert_actions_torch(), env.expert_actions_torch(o))
    env.close()

    # normalize_observations: the policy sees the raw observation, not the normalised one
    raw = make_mt_envs("MT10", seed=1, num_envs=10)
    nrm = make_mt_envs("MT10", seed=1, num_envs=10, normalize_observations=True)
    o_raw, _ = raw.reset(); o_n, _ = nrm.reset()
    assert not np.allclose(o_raw, o_n)
    assert nrm.expert_actions().tobytes() == raw.expert_actions(o_raw).tobytes()
    for _ in range(3):
        a = actions(10)
        o_raw, *_ = raw.step(a); nrm.step(a)
        assert nrm.expert_actions().tobytes() == raw.expert_actions(o_raw).tobytes()
    mt = torch.zeros(10, dtype=torch.bool, device=raw.device); mt[2] = True
    o_raw = raw.reset_torch(mt); nrm.reset_torch(mt)
    assert torch.equal(nrm.expert_actions_torch(), raw.expert_actions_torch(o_raw))
    for _ in range(3):
        a = torch.from_numpy(actions(10)).to(raw.device)
        o_raw, *_ = raw.step_torch(a); nrm.step_torch(a)
        assert torch.equal(nrm.expert_actions_torch(), raw.expert_actions_torch(o_raw))
    raw.close(); nrm.close()

    # NEXT_STEP: the terminal call reports the terminal observation, and so does the default source
    for api in ("numpy", "torch"):
        env = make_mt_envs("MT10", seed=2, num_envs=10, max_episode_steps=4, autoreset_mode="NextStep")
        if api == "numpy":
            env.reset()
        else:
            env.reset_torch()
        ended = False
        for _ in range(6):
            if api == "numpy":
                obs, _, term, trunc, _ = env.step(actions(10))
                ended |= bool((term | trunc).any())
                assert env.expert_actions().tobytes() == env.expert_actions(obs).tobytes()
            else:
                o, _, term, trunc, _ = env.step_torch(torch.from_numpy(actions(10)).to(env.device))
                ended |= bool(((term | trunc) != 0).any())
                assert torch.equal(env.expert_actions_torch(), env.expert_actions_torch(o))
        assert ended
        env.close()


def test_explicit_observation_after_set_state(torch_cuda):
    """An explicit observation (`observe_torch` after `set_state_torch`, one-hot columns included) and argument checks."""
    torch = torch_cuda
    from metaworld_b200.vector_env import make_mt_envs
    env = make_mt_envs("MT10", seed=4, num_envs=10, use_one_hot=True)
    env.reset_torch()
    for _ in range(5):
        env.step_torch(torch.zeros(10, 4, device=env.device))
    qp, qv = env.get_state_torch()
    qp[:, 0] += 0.01                                    # move the arm: a state no step produced
    env.set_state_torch(qp, qv)
    o = env.observe_torch()
    a = env.expert_actions_torch(o)
    assert torch.equal(a, env.expert_actions_torch(o[:, :39].contiguous()))
    assert a.shape == (10, 4) and a.dtype == torch.float32 and torch.isfinite(a).all()
    with pytest.raises(ValueError):
        env.expert_actions_torch(o[:, :30])
    with pytest.raises(ValueError):
        env.expert_actions_torch(o.double())
    env.close()
