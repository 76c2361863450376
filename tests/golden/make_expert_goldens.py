"""Regenerates tests/golden/expert_actions.npz: the reference's scripted policies (`metaworld.policies`) evaluated on the
observations of tests/golden/traj_<task>.npz.

The observation rows are not stored again: `tests/test_policies.py:expert_rows` rebuilds them from the trajectory goldens
(`reset_obs`, `obs`, `p_reset_obs`, `p_obs` (policy-driven, so the later branches of the decision trees are reached),
`po_reset_obs`, `po_obs`, in that order, rounded to float32: what the device kernel reads), about 490 per task.
Per task:
  * `<task>/actions`  float32 [n, 4]: the reference policy's `get_action` on each row widened to float64 (the numpy API's
                      observation), unclipped.
  * `<task>/knife_edge` bool [n]: rows where one of 8 random relative perturbations of size 1e-9 of the observation moves
                      the reference action by more than 1e-5.  These sit on a branch threshold, where the reference's BLAS
                      `dot` inside `np.linalg.norm` may decide differently from an in-order sum.
  * `<task>/rows_sha256`: the SHA-256 of the float32 rows the actions were computed on (the tests check they rebuild
                      the same rows).
`names`: the reference's ENV_POLICY_MAP keys and, in `classes`, their class names.

Run with a Meta-World checkout:  python tests/golden/make_expert_goldens.py /path/to/Metaworld
The policies need numpy only; they are loaded from a bare namespace package (no gymnasium / mujoco import).
"""
import os
import sys
import types
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]   # tests/, the repository root
from test_policies import expert_rows, rows_digest  # noqa: E402

OUT = os.path.join(HERE, "expert_actions.npz")
N_PERTURB, PERTURB, KNIFE_TOL = 8, 1e-9, 1e-5


def policy_map(reference_root):
    if "metaworld" not in sys.modules:
        pkg = types.ModuleType("metaworld")
        pkg.__path__ = [os.path.join(reference_root, "metaworld")]
        sys.modules["metaworld"] = pkg
    import metaworld.policies as MP
    return MP.ENV_POLICY_MAP


def main(reference_root):
    warnings.simplefilter("ignore")
    pmap = policy_map(reference_root)
    rng = np.random.default_rng(7)
    out = {"names": np.array(list(pmap)), "classes": np.array([c.__name__ for c in pmap.values()])}
    for task, cls in pmap.items():
        pol = cls()
        obs = expert_rows(task)
        # (a copy per call: some reference policies write into slices of their input)
        act = np.stack([pol.get_action(o.astype(np.float64).copy()) for o in obs]).astype(np.float32)
        knife = np.zeros(len(obs), dtype=bool)
        for i, o in enumerate(obs.astype(np.float64)):
            for _ in range(N_PERTURB):
                q = o * (1.0 + PERTURB * rng.uniform(-1.0, 1.0, size=39))
                if np.abs(pol.get_action(q) - act[i]).max() > KNIFE_TOL:
                    knife[i] = True
                    break
        out[f"{task}/actions"], out[f"{task}/knife_edge"], out[f"{task}/rows_sha256"] = act, knife, np.array(rows_digest(obs))
        print(task, len(obs), "rows,", int(knife.sum()), "knife-edge", flush=True)
    np.savez_compressed(OUT, **out)


if __name__ == "__main__":
    main(sys.argv[1])
