"""CPU checks of the device expert policies (metaworld_b200/csrc/mw_policies.cuh, metaworld.policies restated).

The header is compiled for the host by g++ (tests/devpolicy/shim.cpp) with contraction off, as nvcc builds it with
--fmad=false, so the statements checked here are the ones k_expert runs (tests/test_gpu_policies.py holds the two builds
to identical bits).  Two references:
  * tests/golden/expert_actions.npz: the reference's own policy code on ~490 observations per task, the rows
    `expert_rows` rebuilds from tests/golden/traj_<task>.npz (tests/golden/make_expert_goldens.py);
  * tests/golden/policy_actions.npz: the reference's policies driving the oracle closed loop (make_policy_goldens.py).
    Driving the oracle with the restated policies must reproduce that run action for action."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

from builds import host_shim

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
# the observation rows of the expert-action fixture, in this order: resets and 60-step random-action rollouts, the
# policy-driven rollouts (they reach the later branches of the decision trees), the partially observable rollout
EXPERT_SOURCES = ("reset_obs", "obs", "p_reset_obs", "p_obs", "po_reset_obs", "po_obs")
# every observation of a trajectory golden, the 500-step episode included (no reference actions needed: kernel vs host)
ALL_SOURCES = EXPERT_SOURCES + ("l_reset_obs", "l_obs")


def build_shim(path):
    """The host build of mw_policies.cuh at `path`, rebuilt when a source is newer."""
    return host_shim("devpolicy", path, headers=("mw_policies.cuh", "mw_task_ids.h"))


def expert_rows(task, sources=EXPERT_SOURCES):
    """float32 [n, 39]: the observations of tests/golden/traj_<task>.npz named by `sources`, rounded to float32 (what the
    device kernel reads)."""
    g = np.load(os.path.join(GOLD, f"traj_{task}.npz"))
    return np.concatenate([g[k].reshape(-1, 39) for k in sources]).astype(np.float32)


def rows_digest(rows):
    return hashlib.sha256(np.ascontiguousarray(rows, dtype=np.float32).tobytes()).hexdigest()


def host_actions(lib, task_ids, obs):
    """The host build's actions float32 [n, 4] for float64 observations [n, >= 39]."""
    o = np.ascontiguousarray(obs, dtype=np.float64)
    ids = np.ascontiguousarray(task_ids, dtype=np.int32)
    out = np.zeros((len(o), 4), dtype=np.float32)
    lib.host_expert_actions(C.c_void_p(ids.ctypes.data), C.c_void_p(o.ctypes.data), C.c_int(o.shape[1]), C.c_int(len(o)),
                            C.c_void_p(out.ctypes.data))
    return out


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return build_shim(str(tmp_path_factory.mktemp("devpolicy") / "libdevpolicy.so"))


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLD, "expert_actions.npz"))


def _tasks():
    from metaworld_b200.tasks import TASK_IDS
    return sorted(TASK_IDS)


def test_policy_map_has_the_reference_names(golden):
    from metaworld_b200 import policies
    assert {k: v.__name__ for k, v in policies.ENV_POLICY_MAP.items()} == dict(zip(golden["names"], golden["classes"]))
    for cls in policies.ENV_POLICY_MAP.values():
        assert getattr(policies, cls.__name__) is cls


@pytest.mark.parametrize("task", _tasks())
def test_host_build_matches_reference_policy(shim, golden, task):
    from metaworld_b200.tasks import TASK_IDS
    obs, ref, knife = expert_rows(task), golden[f"{task}/actions"], golden[f"{task}/knife_edge"]
    assert str(golden[f"{task}/rows_sha256"]) == rows_digest(obs), "fixture rows differ from the trajectory goldens"
    assert len(obs) == len(ref) >= 450 and knife.mean() < 1e-3
    a = host_actions(shim, np.full(len(obs), TASK_IDS[task]), obs.astype(np.float64))
    assert np.isfinite(a).all()
    np.testing.assert_allclose(a[~knife], ref[~knife], rtol=1e-6, atol=1e-6)


def test_unknown_task_id_gives_nan(shim):
    a = host_actions(shim, [-1, 50, 0], np.zeros((3, 39)))
    assert np.isnan(a[:2]).all() and np.isfinite(a[2]).all()


@pytest.mark.parametrize("task", _tasks())
def test_closed_loop_on_oracle_reproduces_reference_run(shim, task):
    """The restated policy drives the oracle env closed loop (clipped to [-1, 1], as the recorder did) on the 5 goals of
    policy_actions.npz: every action equals the recorded one to 1e-6, and each episode ends at the recorded step with
    the recorded success flag."""
    from oracle.tasks import TASKS
    from metaworld_b200 import benchmarks as B
    from metaworld_b200.tasks import TASK_IDS
    g = np.load(os.path.join(GOLD, "policy_actions.npz"))
    acts, lens, succ = g[f"{task}/actions"], g[f"{task}/len"], g[f"{task}/success"]
    tid = np.array([TASK_IDS[task]])
    k0 = 0
    for k, tk in enumerate(B.make_tasks([task], False, seed=42, n_goals=5)):
        env = TASKS[task]()
        env.set_task_vec(tk.unpack()["rand_vec"], False)
        obs, _ = env.reset()
        ok = False
        for t in range(500):
            a = np.clip(host_actions(shim, tid, obs[None])[0], -1, 1)
            assert t < lens[k] and np.abs(a - acts[k0 + t]).max() <= 1e-6, (task, k, t)
            obs, _, _, _, info = env.step(a)
            if info["success"]:
                ok = True
                break
        assert t + 1 == lens[k] and ok == succ[k], (task, k)
        k0 += lens[k]
