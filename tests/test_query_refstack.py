"""The state getters of the bare env and of the vector env's `call` / `get_attr` against the reference's own classes.
The REAL host code runs on tests/oracle_query_engine.py (the float64 oracle behind `Engine.query`); the reference side
is replayed from tests/golden/refstack_<test>.pkl.gz (tests/refstack_replay.py); with METAWORLD_REFERENCE=<Meta-World
checkout> it runs live and rewrites those files."""
import copy

import numpy as np
import pytest

from oracle_query_engine import OracleQueryEngine
from refstack_replay import RefSession

ATOL = 2e-6
_HLO, _HHI = np.array([-0.525, 0.348, -0.0525]), np.array([0.525, 1.025, 0.7])


class _SnapshotSession(RefSession):
    """RefSession that copies each recorded value when it is logged: the getters return views of the reference's MjData
    (data.body(..).xpos), whose memory later steps overwrite before the log is written."""

    def access(self, op, path, args, live):
        n = len(self.log) if self.recording else 0
        try:
            return super().access(op, path, args, live)
        finally:
            if self.recording and len(self.log) > n:
                self.log[-1] = copy.deepcopy(self.log[-1])


@pytest.fixture
def ref(request):
    s = _SnapshotSession(request.node.name.replace("[", "_").rstrip("]"))
    yield s
    s.close()


@pytest.fixture
def metaworld(ref):
    ref.module("gymnasium")
    return ref.module("metaworld")


def _outcome(fn):
    """A getter's value, or the name of the exception it raises."""
    try:
        return "value", fn()
    except Exception as e:      # noqa: BLE001 -- the reference's exception is part of its behaviour
        return "raise", type(e).__name__


def _same(a, b, what):
    assert a[0] == b[0], (what, a, b)
    if a[0] == "raise":
        assert a[1] == b[1], (what, a, b)
        return
    x, y = a[1], b[1]
    if isinstance(x, dict):
        assert set(x) == set(y), what
        for k in x:
            _same(("value", x[k]), ("value", y[k]), (what, k))
    elif x is None or isinstance(x, (bool, np.bool_, int, np.integer)):
        assert x == y and type(bool(x)) is type(bool(y)), (what, x, y)
    else:
        x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
        assert x.shape == y.shape and np.abs(x - y).max() < ATOL, (what, x, y)


_GETTERS = [
    ("get_endeff_pos", lambda e: e.get_endeff_pos()),
    ("tcp_center", lambda e: e.tcp_center),
    ("_get_pos_objects", lambda e: e._get_pos_objects()),
    ("_get_quat_objects", lambda e: e._get_quat_objects()),
    ("_get_pos_goal", lambda e: e._get_pos_goal()),
    ("_target_pos", lambda e: e._target_pos),
    ("obj_init_pos", lambda e: e.obj_init_pos),
    ("init_tcp", lambda e: e.init_tcp),
    ("init_left_pad", lambda e: e.init_left_pad),
    ("init_right_pad", lambda e: e.init_right_pad),
    ("goal site", lambda e: e._get_site_pos("goal")),
    ("rightEndEffector site", lambda e: e._get_site_pos("rightEndEffector")),
    ("missing site", lambda e: e._get_site_pos("no_such_site")),
    ("hand body", lambda e: e.get_body_com("hand")),
    ("_get_id_main_object", lambda e: e._get_id_main_object()),
    ("touching_main_object", lambda e: e.touching_main_object),
    ("touching_object(leftpad)", lambda e: e.touching_object(0)),
]


def _compare(renv, oenv, when, task):
    from metaworld_b200.tasks import MOVED_SITES
    for site in MOVED_SITES.get(task, {}):             # sites reset_model placed through model.site(name).pos
        _same(_outcome(lambda: renv._get_site_pos(site)), _outcome(lambda: oenv._get_site_pos(site)), (when, site))
    for name, fn in _GETTERS:
        a, b = _outcome(lambda: fn(renv)), _outcome(lambda: fn(oenv))
        if a == ("raise", "ValueError") and b == ("raise", "KeyError"):
            continue                    # a missing name: MuJoCo raises KeyError, the bindings the logs were recorded on ValueError
        _same(a, b, (when, name))
    d1, d2 = renv._get_obs_dict(), oenv._get_obs_dict()          # commits the frame stack on both sides
    _same(("value", d1), ("value", d2), (when, "_get_obs_dict"))


@pytest.mark.parametrize("name", ["reach-v3", "push-v3", "hammer-v3", "stick-push-v3", "drawer-close-v3", "basketball-v3",
                                  "shelf-place-v3", "door-lock-v3", "button-press-v3", "assembly-v3", "plate-slide-back-side-v3",
                                  "disassemble-v3", "faucet-open-v3", "faucet-close-v3", "coffee-push-v3"])
def test_bare_env_getters_match_reference_class(metaworld, name):
    """`mt1.train_classes[name]()` and SawyerXYZEnvB200 from the same task and actions: every getter (value, shape,
    exception) mid-episode, after set_state and (reach) after the truncation at 500 steps; the observation's hand and
    object slots equal the getters (tests/helpers.py step_env).  Each comparison point uses its own pair of envs."""
    from metaworld_b200 import benchmarks as B
    from metaworld_b200.single_env import SawyerXYZEnvB200
    metaworld._N_GOALS = 2
    rb, ob = metaworld.MT1(name, seed=3), B.MT1(name, seed=3, n_goals=2)

    def run(steps, then_set_state, when):
        renv = rb.train_classes[name]()
        oenv = SawyerXYZEnvB200(name, engine=OracleQueryEngine([name]))
        renv.set_task(rb.train_tasks[1]); oenv.set_task(ob.train_tasks[1])
        o1, _ = renv.reset(); o2, _ = oenv.reset()
        assert np.abs(o1 - o2).max() < ATOL
        rng = np.random.default_rng(5)
        for t in range(steps):
            a = rng.uniform(-1, 1, size=4).astype(np.float32)
            r1, r2 = renv.step(a.copy()), oenv.step(a.copy())
            assert np.abs(r1[0] - r2[0]).max() < 1e-5 and r1[3] == r2[3], t
        nxt = r2[0]                                                  # step_env's equalities on this package
        assert (nxt[:3] == np.clip(oenv.get_endeff_pos(), _HLO, _HHI)).all()
        assert (nxt[4:7] == oenv._get_pos_objects()[:3]).all() and (nxt[7:11] == oenv._get_quat_objects()[:4]).all()
        if then_set_state:
            qpos, qvel = oenv.get_env_state()
            qpos = qpos + 0.002 * (np.arange(len(qpos)) < 9)
            renv.set_state(qpos.copy(), qvel.copy()); oenv.set_state(qpos.copy(), qvel.copy())
        _compare(renv, oenv, when, name)
        oenv.close()

    run(3, False, "mid-episode")
    run(3, True, "set_state")
    if name == "reach-v3":
        run(500, False, "after the truncation")
