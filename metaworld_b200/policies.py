"""The 50 scripted expert policies of the reference's `metaworld.policies`, computed on the device.

`ENV_POLICY_MAP` has the reference's keys and each class its name (`SawyerPickPlaceV3Policy`, ...).  `get_action(obs)`
takes one 39-column observation and returns the float32 action the reference policy returns for it, unclipped; the
decision logic runs in the CUDA kernel `k_expert` (csrc/mw_policies.cuh), which computes in float64 from the float32
observation, as the reference does on what the numpy vector env hands it.  Importing this module needs neither
gymnasium nor mujoco.

Batched forms: `Policy.get_actions(obs)` ([n, >= 39] numpy rows of one task), module-level `get_actions(obs, tasks)`
(a task name per row) and `MetaWorldVecEnv.expert_actions_torch()` (device tensors, no host synchronisation).

Differences from the reference:
  * the policies read the first 39 columns only, so observations with one-hot task columns work (`get_actions`);
  * an observation is rounded to float32 before the policy sees it (exact for what the environments return);
  * only `Policy.get_action` emits move()'s UserWarning for an action component beyond [-1, 1]; the batched forms are
    silent;
  * action noise is the caller's: `a + sigma * torch.randn_like(a)`.
"""
from __future__ import annotations

import warnings

import numpy as np

from .tasks import TASK_IDS

# move()'s warning text, so that existing warning filters match
_MOVE_WARNING = "Constant(s) may be too high. Environments clip response to [-1, 1]"


def _device():
    import torch
    return torch.device("cuda", torch.cuda.current_device())


def _task_id(name):
    if name not in TASK_IDS:
        raise KeyError(f"no scripted policy for task {name!r}")
    return TASK_IDS[name]


def get_actions(obs, tasks):
    """Expert actions for a batch: `obs` numpy [n, >= 39] (columns past 39, e.g. one-hot ids, are ignored), `tasks` a
    task name for every row or one name for all.  Returns float32 [n, 4], unclipped."""
    import torch

    from .engine import expert_actions
    o = np.asarray(obs)
    if o.ndim != 2 or o.shape[1] < 39:
        raise ValueError(f"get_actions needs observations of shape [n, >= 39], got {o.shape}")
    n = o.shape[0]
    ids = np.full(n, _task_id(tasks), np.int32) if isinstance(tasks, str) else np.array([_task_id(t) for t in tasks], np.int32)
    if ids.shape != (n,):
        raise ValueError(f"get_actions needs one task per observation row ({n}), got {ids.shape[0]}")
    dev = _device()
    d_obs = torch.from_numpy(np.ascontiguousarray(o[:, :39], dtype=np.float32)).to(dev)
    d_ids = torch.from_numpy(ids).to(dev)
    out = torch.empty(n, 4, dtype=torch.float32, device=dev)
    expert_actions(d_ids, d_obs, out)
    return out.cpu().numpy()


class Policy:
    """A scripted expert policy of one task (`task_name`); the base of the 50 classes of `ENV_POLICY_MAP`."""

    task_name: str = ""

    def get_action(self, obs):
        """obs: numpy [39] -> float32 [4] (the reference's `get_action`)."""
        o = np.asarray(obs)
        assert o.ndim == 1 and o.shape[0] == 39, "Observation not fully parsed"
        a = get_actions(o[None], self.task_name)[0]
        if np.any(np.abs(a[:3]) > 1.0):
            warnings.warn(_MOVE_WARNING)
        return a

    def get_actions(self, obs):
        """obs: numpy [n, >= 39] -> float32 [n, 4]."""
        return get_actions(obs, self.task_name)


def _class_name(task):
    # the reference names each class after its task, except that peg-insert-side's says "Insertion"
    stem = "peg-insertion-side" if task == "peg-insert-side-v3" else task[:-3]
    return "Sawyer" + "".join(w.capitalize() for w in stem.split("-")) + "V3Policy"


ENV_POLICY_MAP: dict = {}
for _name in sorted(TASK_IDS):
    _cls = type(_class_name(_name), (Policy,), {"task_name": _name, "__module__": __name__,
                                                "__doc__": f"The scripted expert policy of {_name}."})
    ENV_POLICY_MAP[_name] = _cls
    globals()[_cls.__name__] = _cls
del _name, _cls

__all__ = ["ENV_POLICY_MAP", "Policy", "get_actions"] + [c.__name__ for c in ENV_POLICY_MAP.values()]
