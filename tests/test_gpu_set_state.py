"""GPU suite (-m gpu): setting and reading the physics state on the device (k_set_physics, k_get_physics, k_observe) and
what the vector env builds on them (set_state_torch, get_state_torch, observe_torch)."""
import os

import numpy as np
import pytest

from rig import GOLD, SENSITIVE_OPEN_LOOP, TOL, Rig, _params, steady_mt50
from rig import torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu


def test_setting_every_env_to_its_own_state_changes_nothing(torch_cuda):
    """MT50 @ 4096 in steady state: set_state_torch(*get_state_torch()) on all envs, then 50 steps (autoresets included):
    every step's outputs and the final device records are bitwise those of the same run without the call."""
    torch = torch_cuda
    env = steady_mt50(torch)
    st0 = env.engine.get_state()
    A = torch.from_numpy(np.random.default_rng(7).uniform(-1, 1, size=(50, env.num_envs, 4)).astype(np.float32)).to(env.device)

    def run(roundtrip):
        env.engine.set_state(st0)
        if roundtrip:
            env.set_state_torch(*env.get_state_torch())
        out = []
        for t in range(50):
            out.append([x.clone() for x in env.step_torch(A[t])])
        return out, env.engine.get_state()

    ref, st_ref = run(False)
    got, st_got = run(True)
    assert all(torch.equal(x, y) for a, b in zip(ref, got) for x, y in zip(a, b))
    assert st_ref.tobytes() == st_got.tobytes()
    assert sum(int(a[3].sum()) for a in ref) > 100                 # truncations (and restarts) inside the window
    assert not env.engine.faults().any()
    env.close()


@pytest.mark.parametrize("mode", ["SameStep", "NextStep", "Disabled"])
def test_branches_copied_from_one_env_stay_bitwise_equal(torch_cuda, mode):
    """64 envs of one task and goal, reset together, step with different actions; env 0's qpos / qvel is copied into all
    of them, observe_torch commits the frame stack, and the same actions follow: every row equals env 0's, bit for bit,
    up to and including the step that ends the episode.  set_state leaves the mocap target and the solver's warm-start
    acceleration alone (as the reference's does), and both steer the next step, so the test first gives every env env 0's
    through the raw record: the branches then differ only in what set_state and observe overwrite."""
    torch = torch_cuda
    from metaworld_b200 import benchmarks as B
    from metaworld_b200.vector_env import MetaWorldVecEnv
    name, n, M, k = "pick-place-v3", 64, 30, 12
    task = B.MT1(name, seed=3).train_tasks[0]
    env = MetaWorldVecEnv([name] * n, [[task]] * n, seed=3, max_episode_steps=M, autoreset_mode=mode)
    dev = env.device
    env.reset_torch()
    rng = np.random.default_rng(1)
    for _ in range(k):
        a = rng.uniform(-1, 1, size=(n, 4)).astype(np.float32)
        a[:, 3] = np.where(np.arange(n) % 2 == 0, 1.0, a[:, 3])
        env.step_torch(torch.from_numpy(a).to(dev))
    st = env.engine.get_state()
    for f in ("warm", "mocap_pos"):
        st[f] = st[f][0]
    env.engine.set_state(st)
    qpos, qvel = env.get_state_torch()
    assert not torch.equal(qpos[1], qpos[0])
    env.set_state_torch(qpos[:1].expand(n, -1).contiguous(), qvel[:1].expand(n, -1).contiguous())
    o = env.observe_torch()
    assert torch.equal(o[:, :18], o[:1, :18].expand(n, -1)) and torch.equal(o[:, 36:], o[:1, 36:].expand(n, -1))
    rec = env.engine.get_state()
    assert all(rec[f].tobytes() == np.repeat(rec[f][:1], n, 0).tobytes() for f in ("qpos", "qvel", "warm", "mocap_pos", "prev_obs"))
    ended_at = None
    for t in range(k, M + 2):
        a = np.repeat(rng.uniform(-1, 1, size=(1, 4)).astype(np.float32), n, 0)
        out = env.step_torch(torch.from_numpy(a).to(dev))
        for x in out:
            assert torch.equal(x, x[:1].expand_as(x)), (mode, t)
        if bool(out[2][0] | out[3][0]):
            ended_at = t
            break
    assert ended_at == M - 1
    assert not env.engine.faults().any()
    env.close()


@pytest.mark.parametrize("task", _params(SENSITIVE_OPEN_LOOP))
def test_set_state_observe_and_steps_match_the_oracle(torch_cuda, task):
    """A mid-episode state of one goal's golden trajectory set into an env running another goal: observe equals the
    oracle's set_state + _get_obs() to 1e-5, and 20 steps after it agree with the oracle to 1e-4 (obs, reward, 7 infos)."""
    torch = torch_cuda
    from oracle.tasks import TASKS as OT
    g = np.load(os.path.join(GOLD, f"traj_{task}.npz"))
    rig = Rig(torch, task, g["rand_vec"][1:2])
    rig.reset()
    oracle = OT[task]()
    lo, _ = oracle.random_reset_space()
    oracle.set_task_vec(g["rand_vec"][1][: len(lo)], False)
    oracle.reset()
    A = g["actions"][0]
    for t in range(3):
        rig.step(A[t:t + 1]); oracle.step(A[t])
    nq, nv = g["qpos"].shape[2], g["qvel"].shape[2]
    qpos = np.zeros((1, 18)); qpos[0, :nq] = g["qpos"][0, 30]
    qvel = np.zeros((1, 17)); qvel[0, :nv] = g["qvel"][0, 30].astype(np.float32)   # the record keeps qvel in float32
    d = rig.eng.device
    mask = torch.ones(1, dtype=torch.bool, device=d)
    rig.eng.set_physics(mask, torch.from_numpy(qpos).to(d), torch.from_numpy(qvel).to(d))
    out = torch.zeros(1, 39, device=d)
    rig.eng.observe(mask, out)
    oracle.set_state(qpos[0, :nq].copy(), qvel[0, :nv].copy())
    err_obs0 = np.abs(out[0].cpu().numpy() - oracle._get_obs()).max()
    worst_o = worst_r = worst_i = 0.0
    for t in range(31, 51):
        o, r, info, _, _ = rig.step(A[t:t + 1])
        oo, orw, _, _, oi = oracle.step(A[t])
        worst_o = max(worst_o, np.abs(o[0] - oo).max())
        worst_r = max(worst_r, abs(r[0] - orw))
        worst_i = max(worst_i, max(abs(info[0, i] - float(oi[key])) for i, key in enumerate(
            ("success", "near_object", "grasp_success", "grasp_reward", "in_place_reward", "obj_to_target", "unscaled_reward"))))
    print(f"{task}: observe err {err_obs0:.2e}; 20 steps worst obs {worst_o:.2e} reward {worst_r:.2e} info {worst_i:.2e}")
    assert err_obs0 < 1e-5
    assert worst_o < TOL and worst_r < TOL and worst_i < TOL


def test_masked_calls_leave_the_other_rows_alone(torch_cuda):
    """MT10 @ 700: set_state_torch / observe_torch with a mask change the masked envs' records and observation rows only;
    no fault bit is set."""
    torch = torch_cuda
    from metaworld_b200.vector_env import make_mt_envs
    env = make_mt_envs("MT10", seed=9, num_envs=700, use_one_hot=True)
    dev = env.device
    env.reset_torch()
    rng = np.random.default_rng(2)
    for _ in range(6):
        env.step_torch(torch.from_numpy(rng.uniform(-1, 1, size=(700, 4)).astype(np.float32)).to(dev))
    mask_np = rng.random(700) < 0.3
    mask = torch.from_numpy(mask_np).to(dev)
    obs0 = env.observe_torch().clone()
    st0 = env.engine.get_state()
    qpos, qvel = env.get_state_torch()
    q2, v2 = qpos.clone(), qvel.clone()
    q2[:, :7] += 0.05; v2[:, :7] += 0.1                        # arm joints of every model
    env.set_state_torch(q2, v2, env_mask=mask)
    obs1 = env.observe_torch(mask).clone()
    st1 = env.engine.get_state()
    keep, hit = ~mask_np, mask_np
    assert st1[keep].tobytes() == st0[keep].tobytes()
    assert torch.equal(obs1[torch.from_numpy(keep).to(dev)], obs0[torch.from_numpy(keep).to(dev)])
    assert (st1["qpos"][hit, :7] != st0["qpos"][hit, :7]).all() and (st1["prev_obs"][hit] != st0["prev_obs"][hit]).any(axis=1).all()
    for f in ("warm", "mocap_pos", "target", "path_len", "episode", "ep_return", "snapshot", "scal", "obj_init"):
        assert st1[f][hit].tobytes() == st0[f][hit].tobytes(), f
    q, v = env.get_state_torch()
    assert torch.equal(q[mask][:, :7], q2[mask][:, :7]) and torch.equal(v[mask][:, :7], v2[mask][:, :7].float().double())
    assert not env.engine.faults().any()
    with pytest.raises(ValueError):
        env.set_state_torch(q2.float(), v2)
    with pytest.raises(ValueError):
        env.observe_torch(mask.cpu())
    env.close()
