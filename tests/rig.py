"""What the GPU tests (tests/test_gpu*.py) and scripts/gpu_diag.py share: the `torch_cuda` fixture, random actions and
the DISABLED restarts of the vector env (`acts`, `reset_ended`), its steady-state MT50 setup (`steady_mt50`), the golden
trajectories, the tolerance, the known float32-vs-float64 sensitivities, and `Rig`, N envs of one task on the raw
engine.  A test module takes the fixture with `from rig import torch_cuda`."""
import glob
import os

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-4


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch


def acts(torch, rng, n, dev):
    return torch.from_numpy(rng.uniform(-1, 1, size=(n, 4)).astype(np.float32)).to(dev)


def reset_ended(env, out):
    """DISABLED autoreset: restart the envs whose episode ended in this step; returns the reset observation (or None)."""
    if env.autoreset_mode != "Disabled":
        return None
    return env.reset_torch(env.torch.logical_or(out[2], out[3]).bool()).clone()


def steady_mt50(torch, mode="SameStep", n=4096, seed=42):
    """MT50 with one-hot ids in `mode`, episode phases spread over 0..499 by bench.py's `stagger`, 20 steps in."""
    import bench
    from metaworld_b200.vector_env import make_mt_envs
    env = make_mt_envs("MT50", seed=seed, num_envs=n, use_one_hot=True, autoreset_mode=mode)
    env.reset_torch()
    bench.stagger(env, seed)
    rng = np.random.default_rng(seed + 1)
    for _ in range(20):
        reset_ended(env, env.step_torch(acts(torch, rng, n, env.device)))
    return env


def _tasks_with_goldens():
    from metaworld_b200.tasks import TASKS
    names = [os.path.basename(p)[5:-4] for p in sorted(glob.glob(os.path.join(GOLD, "traj_*.npz")))]
    return [n for n in names if n in TASKS]


# Known float32-vs-float64 sensitivities (measured, see DESIGN.md section 7).  These are
# reported as xfail with the reason, never skipped: each one is a place where contact dynamics amplify a 1e-7 state
# difference (an object jammed in a hole, a nut resting on a peg, an object that starts exactly touching a surface so
# that `dist < margin` is decided by the last bit), not a missing feature.
_JAMMED = "resting contacts under load are chaotic: float32 step vs float64 oracle diverge beyond 1e-4 within the rollout"
_TOUCH = "object starts exactly touching (dist == margin to the last bit): contact inclusion differs between float32 and float64 state"
SENSITIVE_RESET = {"disassemble-v3": _JAMMED, "peg-unplug-side-v3": _JAMMED}
SENSITIVE_OPEN_LOOP = {"assembly-v3": _JAMMED, "basketball-v3": _TOUCH, "box-close-v3": _JAMMED, "coffee-push-v3": _JAMMED,
                       "disassemble-v3": _JAMMED,
                       "peg-unplug-side-v3": "the plug starts jammed in its socket (SENSITIVE_RESET): the rollout amplifies any change of float32 rounding "
                                             "(e.g. a different FMA contraction after a refactor) to ~3e-4 within 60 steps; single steps agree to 3e-5 (contact-rich test)",
                       "handle-press-v3": "observations agree to 3e-6; the reward (slope ~50 near the handle) turns that into 1.4e-4",
                       "drawer-close-v3": "goal 0's golden trajectory passes 1.07e-7 m from a contact-activation discontinuity (the left claw grazes the drawer front inside the "
                                          "1 mm margin at step 2): the float64 oracle itself jumps by 1.08e-4 when the drawer is moved by 1.08e-7 "
                                          "(tests/test_oracle.py::test_drawer_close_golden_knife_edge); float32 state noise puts the device on the other side"}
SENSITIVE_ONE_STEP = {"assembly-v3": "the nut rests on the peg (mesh-cylinder contacts under load): single steps reach 1.2e-4"}
SENSITIVE_CONTACT_RICH = {"soccer-v3": "mesh-mesh face contact (hand against the goal frame): EPA witness point on a flat patch is path dependent"}


def _report(name, row):
    """Appends one measurement row to $MW_TEST_REPORT_DIR/<name> when that variable names a directory to collect them in."""
    d = os.environ.get("MW_TEST_REPORT_DIR")
    if d:
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, name), "a") as f:
            f.write(row)


def _params(sensitive):
    return [pytest.param(t, marks=pytest.mark.xfail(reason=sensitive[t], strict=False)) if t in sensitive else t
            for t in _tasks_with_goldens()]


# the tasks whose reference policy fails on the reference glue itself (test_scripted_policy_actions_succeed and the
# closed-loop policy tests of tests/test_gpu_policies.py)
POLICY_FAILS_ON_REFERENCE_GLUE = {"basketball-v3": "the reference's own policy scores 0/5 on the reference glue (DESIGN.md section 8: target aliasing)",
                                  "peg-insert-side-v3": "the reference's own policy scores 3/5 on the reference glue with these goals"}


class Rig:
    """N envs of one task, driven through the raw engine (C ABI)."""

    def __init__(self, torch, task, rand_vecs, partial=False):
        from metaworld_b200.engine import Engine
        self.t = torch
        self.eng = Engine([task])
        n = len(rand_vecs)
        self.ids = self.eng.build_snapshots([0] * n, rand_vecs, [int(partial)] * n)
        self.eng.set_envs([0] * n)
        self.eng.set_options(500, False, 0)
        d = self.eng.device
        self.n = n
        self.obs = torch.zeros(n, 39, device=d); self.rew = torch.zeros(n, device=d)
        self.term = torch.zeros(n, dtype=torch.uint8, device=d); self.trunc = torch.zeros(n, dtype=torch.uint8, device=d)
        self.info = torch.zeros(n, 7, device=d); self.fobs = torch.zeros(n, 39, device=d); self.finfo = torch.zeros(n, 8, device=d)
        self.sid = torch.tensor(self.ids, dtype=torch.int32, device=d)

    def reset(self):
        self.eng.reset(self.sid, self.obs)
        return self.obs.cpu().numpy()

    def step(self, a):
        self.eng.step(self.t.tensor(np.ascontiguousarray(a, dtype=np.float32), device=self.eng.device), self.obs, self.rew, self.term,
                      self.trunc, self.info, self.fobs, self.finfo, self.sid)
        return self.obs.cpu().numpy(), self.rew.cpu().numpy(), self.info.cpu().numpy(), self.term.cpu().numpy(), self.trunc.cpu().numpy()

    def load_golden(self, g, t, pre=""):
        """Sets every env's record to state t of the golden `g` (tests/golden/traj_<task>.npz; pre="p_" for the policy
        trajectory): qpos, qvel, mocap, the previous observation, a zero warm start, path_len t + 1."""
        nq, nv = g[pre + "qpos"].shape[2], g[pre + "qvel"].shape[2]
        st = self.eng.get_state()
        for k in range(self.n):
            st[k]["qpos"][:nq] = g[pre + "qpos"][k, t]; st[k]["qvel"][:nv] = g[pre + "qvel"][k, t]
            st[k]["mocap_pos"] = g[pre + "mocap"][k, t]; st[k]["prev_obs"] = g[pre + "obs"][k, t][:18]
            st[k]["warm"][:] = 0; st[k]["path_len"] = t + 1
        self.eng.set_state(st)
