"""GPU suite (-m gpu): the read-only state query on the device (k_query / mw_query) and the accessors built on it
(query_torch, the reference's getters through call / get_attr and on the bare env)."""
import os

import numpy as np
import pytest

from test_gpu import GOLD, Rig, _tasks_with_goldens
from test_gpu_set_state import _steady_mt50

pytestmark = pytest.mark.gpu

_HLO = np.array([-0.525, 0.348, -0.0525], dtype=np.float32)     # SawyerXYZEnv._HAND_SPACE
_HHI = np.array([0.525, 1.025, 0.7], dtype=np.float32)


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch


def _actions(torch, env, steps, seed=7):
    return torch.from_numpy(np.random.default_rng(seed).uniform(-1, 1, size=(steps, env.num_envs, 4)).astype(np.float32)).to(env.device)


def test_frame_is_bitwise_the_step_observation(torch_cuda):
    """MT50 @ 4096 in steady state, 30 steps with autoresets: after every step the queried frame equals the step's
    obs[:, :18], bitwise on the unclipped columns 3..17 and after the hand-space clip on columns 0..2."""
    torch = torch_cuda
    env = _steady_mt50(torch)
    A = _actions(torch, env, 30)
    lo, hi = torch.from_numpy(_HLO).to(env.device), torch.from_numpy(_HHI).to(env.device)
    for t in range(30):
        obs, _, term, trunc, _ = env.step_torch(A[t])
        fr = env.query_torch()["frame"]
        # a row whose episode ended reports its restart snapshot's observation, which the float64 build computed
        keep = ~(term.bool() | trunc.bool())
        assert int(keep.sum()) > env.num_envs // 2
        assert torch.equal(fr[keep, 3:], obs[keep, 3:18]), t
        assert torch.equal(torch.minimum(torch.maximum(fr[keep, :3], lo), hi), obs[keep, :3]), t
    assert not env.engine.faults().any()
    env.close()


def test_query_has_no_side_effects(torch_cuda):
    """The same 30 steps with and without a full query (16 named frames and touching) between them: bitwise equal step
    outputs and final device records, and no fault bit."""
    torch = torch_cuda
    env = _steady_mt50(torch)
    st0 = env.engine.get_state()
    A = _actions(torch, env, 30)
    bodies = ("hand", "rightpad", "leftpad", "obj", "rightclaw", "leftclaw")
    sites = ("rightEndEffector", "leftEndEffector", "goal", "hole", "handle")
    geoms = ("objGeom", "leftpad_geom", "rightpad_geom", "handle", "mug")

    def run(query):
        env.engine.set_state(st0)
        out = []
        for t in range(30):
            out.append([x.clone() for x in env.step_torch(A[t])])
            if query:
                q = env.query_torch(bodies=bodies, sites=sites, geoms=geoms, touching=True)
                assert q["body_xpos"].shape == (env.num_envs, 6, 3) and q["site_xmat"].shape == (env.num_envs, 5, 3, 3)
        return out, env.engine.get_state()

    ref, st_ref = run(False)
    got, st_got = run(True)
    assert all(torch.equal(x, y) for a, b in zip(ref, got) for x, y in zip(a, b))
    assert st_ref.tobytes() == st_got.tobytes()
    assert not env.engine.faults().any()
    env.close()


@pytest.mark.parametrize("task", _tasks_with_goldens())
def test_poses_and_frame_match_the_oracle(torch_cuda, task):
    """A golden qpos row set on both sides: every body, site and geom of the model matches the oracle's
    data.body / site / geom(name) pose to 1e-5, and the frame matches the oracle's first 18 observation columns."""
    torch = torch_cuda
    from oracle.tasks import TASKS as OT
    from metaworld_b200 import modelzoo
    from metaworld_b200.tasks import TASKS
    from metaworld_b200.vector_env import _quat2mat
    g = np.load(os.path.join(GOLD, f"traj_{task}.npz"))
    rig = Rig(torch, task, g["rand_vec"][1:2])
    rig.reset()
    oracle = OT[task]()
    lo, _ = oracle.random_reset_space()
    oracle.set_task_vec(g["rand_vec"][1][: len(lo)], False)
    oracle.reset()
    nq, nv = g["qpos"].shape[2], g["qvel"].shape[2]
    qpos = np.zeros((1, 18)); qpos[0, :nq] = g["qpos"][0, 30]
    qvel = np.zeros((1, 17)); qvel[0, :nv] = g["qvel"][0, 30].astype(np.float32)
    d = rig.eng.device
    mask = torch.ones(1, dtype=torch.bool, device=d)
    rig.eng.set_physics(mask, torch.from_numpy(qpos).to(d), torch.from_numpy(qvel).to(d))
    oracle.set_state(qpos[0, :nq].copy(), qvel[0, :nv].copy())
    names = modelzoo.full_model(TASKS[task].xml).names
    frames = [(k, n) for k in ("body", "site", "geom") for n in names[k] if n]
    frame = torch.zeros(1, 18, device=d)
    pose = torch.zeros(1, len(frames), 7, dtype=torch.float64, device=d)
    rig.eng.query(mask, frame=frame, pose=pose, frames=frames)
    p = pose[0].cpu().numpy()
    R = _quat2mat(pose[0, :, 3:]).cpu().numpy()
    err_frame = np.abs(frame[0].cpu().numpy() - oracle._get_obs()[:18]).max()
    assert err_frame < 1e-5
    errs = []
    for i, (kind, n) in enumerate(frames):
        v = getattr(oracle.data, kind)(n)
        e_pos = np.abs(p[i, :3] - v.xpos).max()
        e_rot = np.abs(R[i].reshape(-1) - np.asarray(v.xmat).reshape(-1)).max()
        errs.append((max(e_pos, e_rot), kind, n, e_pos, e_rot))
    # the oracle leaves the faucet's goal sites where the model file puts them; the reference sets model.site(..).pos
    # to _target_pos (sawyer_faucet_open_v3.py:114, sawyer_faucet_close_v3.py:116), pinned in tests/test_query_refstack.py
    target = rig.eng.get_state()[0]["target"].astype(np.float64)
    for i, (kind, n) in enumerate(frames):
        if (task, n) in (("faucet-open-v3", "goal_open"), ("faucet-close-v3", "goal_close")):
            assert np.abs(p[i, :3] - target).max() < 1e-6
            errs[i] = (0.0,) + errs[i][1:]
    bad = sorted((e for e in errs if e[0] >= 1e-5), reverse=True)
    print(f"{task}: {len(frames)} frames, frame err {err_frame:.2e}, {len(bad)} poses off: {bad[:4]}")
    assert not bad, bad


def test_masked_query_writes_only_masked_rows(torch_cuda):
    """MT10 @ 700 with every third env masked: the other rows of each output keep their sentinel fill."""
    torch = torch_cuda
    from metaworld_b200.vector_env import make_mt_envs
    env = make_mt_envs("MT10", seed=5, num_envs=700)
    env.reset_torch()
    for a in _actions(torch, env, 5):
        env.step_torch(a)
    n, d = env.num_envs, env.device
    mask = torch.from_numpy(np.arange(n) % 3 == 0).to(d)
    frames = [("body", "hand"), ("site", "goal"), ("geom", "objGeom")]
    frame = torch.full((n, 18), 7.0, device=d)
    pose = torch.full((n, 3, 7), 7.0, dtype=torch.float64, device=d)
    touch = torch.full((n,), 7, dtype=torch.uint8, device=d)
    env.engine.query(mask, frame=frame, pose=pose, frames=frames, touching=touch, main_geom=["objGeom"] * 10)
    m = mask.cpu().numpy()
    assert (frame.cpu().numpy()[~m] == 7).all() and (pose.cpu().numpy()[~m] == 7).all() and (touch.cpu().numpy()[~m] == 7).all()
    assert (frame.cpu().numpy()[m] != 7).any(axis=1).all() and (touch.cpu().numpy()[m] <= 1).all()
    full = env.query_torch(bodies=("hand",))
    assert torch.equal(full["frame"][mask], frame[mask]) and torch.equal(full["body_xpos"][mask][:, 0], pose[mask][:, 0, :3])
    assert not env.engine.faults().any()
    env.close()


@pytest.mark.parametrize("task", sorted(__import__("metaworld_b200.tasks", fromlist=["TASKS"]).TASKS))
def test_reference_step_env_on_the_bare_env(torch_cuda, task):
    """The reference's tests/helpers.py step_env (render=False), 100 random steps on SawyerXYZEnvB200: the observation's
    hand, object and goal slots equal the getters exactly."""
    from metaworld_b200 import benchmarks as B
    from metaworld_b200.single_env import SawyerXYZEnvB200
    env = SawyerXYZEnvB200(task)
    env.set_task(B.MT1(task, seed=0).train_tasks[0])
    env.seed(0)
    obs, _ = env.reset()
    for _ in range(100):
        nxt, _, term, trunc, _ = env.step(env.action_space.sample())
        if env._partially_observable:
            assert (nxt[-3:] == np.zeros(3)).all()
        elif task == "basketball-v3":
            # _target_pos aliases the goal site's xpos, which the hoop body carries away from the goal space after the
            # first forward pass; the observation clips it (the reference's own step_env fails here: tests/test_query.py)
            g = env._get_pos_goal()
            assert (nxt[-3:] == np.clip(g, env.goal_space.low, env.goal_space.high).astype(np.float32)).all()
            assert g[2] > env.goal_space.high[2]
        else:
            assert (nxt[-3:] == env._get_pos_goal()).all()
        assert (nxt[:3] == env.get_endeff_pos()).all()
        po, pq = env._get_pos_objects(), env._get_quat_objects()
        assert (nxt[4:7] == po[:3]).all() and (nxt[7:11] == pq[:4]).all()
        if po.shape == (6,):
            assert pq.shape == (8,) and (nxt[11:14] == po[3:]).all() and (nxt[14:18] == pq[4:]).all()
        else:
            assert (nxt[11:14] == 0).all() and (nxt[14:18] == 0).all()
        assert (obs[:18] == nxt[18:-3]).all()
        obs = nxt
        if term or trunc:
            break
    env.close()


def _pad_forces(env, gid):
    """Summed normal forces of the left and right pad contacts with geom `gid` in the oracle's last forward pass."""
    d = env.data
    lid, rid = d.geom("leftpad_geom").id, d.geom("rightpad_geom").id
    lf = rf = 0.0
    for c in d.contact:
        if c.efc_address < 0:
            continue
        pair = (c.geom1, c.geom2)
        if lid in pair and gid in pair:
            lf += d.efc_force[c.efc_address]
        if rid in pair and gid in pair:
            rf += d.efc_force[c.efc_address]
    return lf, rf


def _touching_rows(torch, task):
    from oracle.tasks import TASKS as OT
    from metaworld_b200.tasks import MAIN_OBJECT
    g = np.load(os.path.join(GOLD, f"traj_{task}.npz"))
    rows = [(j, t) for j in range(len(g["p_len"])) for t in range(int(g["p_len"][j]) - 1)]
    rig = Rig(torch, task, np.stack([g["p_rand_vec"][j] for j, _ in rows]))
    rig.reset()
    nq, nv = g["p_qpos"].shape[2], g["p_qvel"].shape[2]
    st = rig.eng.get_state()
    for k, (j, t) in enumerate(rows):
        st[k]["qpos"][:nq] = g["p_qpos"][j, t]
        st[k]["qvel"][:nv] = g["p_qvel"][j, t]
        st[k]["mocap_pos"] = g["p_mocap"][j, t]
        st[k]["warm"] = 0
    rig.eng.set_state(st)
    A = np.stack([g["p_actions"][j, t + 1] for j, t in rows]).astype(np.float32)
    rig.step(A)
    assert (rig.eng.get_state()["gripper_ctrl"] == A[:, 3]).all()
    d = rig.eng.device
    touch = torch.zeros(rig.n, dtype=torch.bool, device=d)
    rig.eng.query(torch.ones(rig.n, dtype=torch.bool, device=d), touching=touch, main_geom=[MAIN_OBJECT[task][0]])
    got = touch.cpu().numpy()
    oracles = {}
    n_true = n_cmp = 0
    for k, (j, t) in enumerate(rows):
        if j not in oracles:
            o = OT[task]()
            lo, _ = o.random_reset_space()
            o.set_task_vec(g["p_rand_vec"][j][: len(lo)], False)
            o.reset()
            oracles[j] = o
        o = oracles[j]
        o.set_state(g["p_qpos"][j, t].copy(), g["p_qvel"][j, t].astype(np.float32).astype(np.float64))
        o.data.mocap_pos[0][:] = g["p_mocap"][j, t]
        o.step(A[k])
        want = bool(o.touching_main_object)
        lf, rf = _pad_forces(o, o._get_id_main_object())
        if (lf > 1e-2 and rf > 1e-2) or (lf == 0 and rf == 0):
            assert got[k] == want, (k, j, t, lf, rf)
            n_cmp += 1
            n_true += want
        else:
            print(f"{task} row {j}/{t}: pad forces {lf:.3g} / {rf:.3g}, device {got[k]}, oracle {want} (not compared)")
    print(f"{task}: {n_cmp} of {len(rows)} rows compared, {n_true} touching")
    return n_true


def test_touching_matches_the_oracle(torch_cuda):
    """Policy-driven golden rows of push, pick-place, coffee-pull, stick-pull and soccer (the fingers close on the
    object): each row's qpos / qvel / mocap target set on both sides, one golden action stepped, then `touching` equals
    the oracle's touching_main_object on every row where the oracle's two pad forces are both above 1e-2 or both zero,
    and at least 20 of those rows touch.  The step writes the gripper command the query drives the fingers with."""
    n_true = sum(_touching_rows(torch_cuda, t) for t in ("push-v3", "pick-place-v3", "coffee-pull-v3", "stick-pull-v3", "soccer-v3"))
    assert n_true >= 20
