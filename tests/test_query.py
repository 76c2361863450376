"""The state getters (query_torch, the reference's SawyerXYZEnv accessors through call / get_attr and on the bare env) with
the real host code on a CPU stand-in of the engine (tests/oracle_query_engine.py), checked against the float64 oracle."""
import numpy as np
import pytest
import torch

from oracle_query_engine import OracleQueryEngine

_HLO, _HHI = np.array([-0.525, 0.348, -0.0525]), np.array([0.525, 1.025, 0.7])


def _vec(name, **kw):
    from metaworld_b200 import benchmarks as B
    from metaworld_b200 import vector_env as V
    names = {"MT10": B.MT10}.get(name, [name])
    return V.make_mt_envs(name, engine=OracleQueryEngine(list(dict.fromkeys(names))), **kw)


def test_query_torch_checks_its_inputs():
    v = _vec("MT10", seed=1, num_goals=2)
    with pytest.raises(RuntimeError):
        v.query_torch()                                              # before reset
    v.reset()
    for bad in (torch.ones(9, dtype=torch.bool), torch.ones(10, dtype=torch.uint8), np.ones(10, dtype=bool)):
        with pytest.raises(ValueError):
            v.query_torch(env_mask=bad)
    for kw in (dict(bodies="hand"), dict(sites=(1,)), dict(geoms=[None])):
        with pytest.raises(ValueError):
            v.query_torch(**kw)
    q = v.query_torch(bodies=("hand", "no_such_body"), sites=("goal",), touching=True)
    assert q["frame"].shape == (10, 18) and q["body_xpos"].shape == (10, 2, 3) and q["body_xquat"].shape == (10, 2, 4)
    assert q["site_xmat"].shape == (10, 1, 3, 3) and q["geom_xpos"].shape == (10, 0, 3) and q["touching"].dtype == torch.bool
    assert torch.isnan(q["body_xpos"][:, 1]).all() and not torch.isnan(q["body_xpos"][:, 0]).any()


def test_step_env_through_call_matches_the_observation():
    """The reference's step_env equalities through the vector env's `call`, on MT10 for 3 steps."""
    v = _vec("MT10", seed=3, num_goals=2)
    obs, _ = v.reset()
    rng = np.random.default_rng(0)
    for _ in range(3):
        nxt, *_ = v.step(rng.uniform(-1, 1, size=(10, 4)).astype(np.float32))
        ee, po, pq = v.call("get_endeff_pos"), v.call("_get_pos_objects"), v.call("_get_quat_objects")
        for e in range(10):
            assert (nxt[e, :3] == np.clip(ee[e], _HLO, _HHI)).all()
            assert (nxt[e, 4:7] == po[e][:3]).all() and (nxt[e, 7:11] == pq[e][:4]).all()
            assert po[e].shape in ((3,), (6,)) and pq[e].shape == (4 + 4 * (po[e].shape == (6,)),)
        assert (obs[:, :18] == nxt[:, 18:36]).all()
        obs = nxt


@pytest.mark.parametrize("name", ["reach-v3", "hammer-v3", "door-lock-v3", "button-press-v3", "basketball-v3",
                                  "shelf-place-v3", "push-v3", "stick-push-v3", "drawer-close-v3"])
def test_bare_env_getters_match_the_oracle(name):
    """SawyerXYZEnvB200's getters against the oracle env driven by the same goal and actions: values, shapes and the
    reference's exceptions, after reset, mid-episode and after set_state."""
    from metaworld_b200 import benchmarks as B
    from metaworld_b200.single_env import SawyerXYZEnvB200
    eng = OracleQueryEngine([name])
    env = SawyerXYZEnvB200(name, engine=eng)
    env.set_task(B.MT1(name, seed=2, n_goals=2).train_tasks[0])
    env.reset()
    ref = eng.envs[0]                                   # the stand-in's own oracle env is the reference here
    rng = np.random.default_rng(1)

    def check():
        assert np.abs(env.get_endeff_pos() - ref.get_endeff_pos()).max() < 1e-6
        assert np.abs(env.tcp_center - ref.tcp_center).max() < 1e-9
        assert np.abs(env.get_body_com("hand") - ref.get_body_com("hand")).max() < 1e-9
        assert np.abs(env._get_site_pos("rightEndEffector") - ref._get_site_pos("rightEndEffector")).max() < 1e-9
        po, pq = env._get_pos_objects(), env._get_quat_objects()
        assert po.dtype == np.float64 and po.shape == np.shape(ref._get_pos_objects()) and pq.shape == np.shape(ref._get_quat_objects())
        assert np.abs(po - ref._get_pos_objects()).max() < 1e-6
        assert np.abs(env.init_tcp - ref.init_tcp).max() < 1e-6
        assert np.abs(env.init_left_pad - ref.init_left_pad).max() < 1e-9
        assert np.abs(env.init_right_pad - ref.init_right_pad).max() < 1e-9
        d = env._get_obs_dict()
        assert set(d) == {"state_observation", "state_desired_goal", "state_achieved_goal"}
        assert d["state_achieved_goal"].shape == ((3,) if name in ("stick-push-v3", "assembly-v3") else (33,))

    check()
    with pytest.raises(KeyError):
        env._get_site_pos("no_such_site")
    with pytest.raises(KeyError):
        env.get_body_com("no_such_body")
    if name in ("door-lock-v3",):
        assert env._get_id_main_object() is None and env.touching_main_object is False
    elif name in ("hammer-v3", "button-press-v3", "basketball-v3"):
        with pytest.raises(AttributeError):
            env._get_id_main_object()
        with pytest.raises(AttributeError):
            env.touching_main_object
    else:
        gid = env._get_id_main_object()
        assert isinstance(gid, int) and env.touching_main_object == ref.touching_main_object
    for t in range(6):
        env.step(rng.uniform(-1, 1, size=4).astype(np.float32))
    check()
    qpos, qvel = env.get_env_state()
    env.set_state(qpos + 0.001 * (np.arange(len(qpos)) < 9), qvel)
    check()
    env.close()


def test_vector_get_attr_and_call_route_the_reference_names():
    v = _vec("MT10", seed=1, num_goals=2)
    v.reset()
    v.step(np.zeros((10, 4), dtype=np.float32))
    for name in ("tcp_center", "_target_pos", "obj_init_pos", "init_tcp", "init_left_pad", "init_right_pad", "hand_init_pos"):
        vals = v.get_attr(name)
        assert len(vals) == 10 and all(np.shape(x) == (3,) for x in vals), name
    goal = v.call("_get_pos_goal")
    assert all((g == t).all() for g, t in zip(goal, v.get_attr("_target_pos")))
    hand = v.call("get_body_com", "hand")
    assert all(np.abs(h - ee).max() < 1e-6 for h, ee in zip(hand, v.call("get_endeff_pos")))
    with pytest.raises(KeyError):
        v.call("_get_site_pos", "no_such_site")
    with pytest.raises(KeyError):                       # the first sub-env that fails: door-open has no objGeom
        v.get_attr("touching_main_object")
    assert len(v.call("touching_object", 0)) == 10
