"""CPU stand-in for the engine's goal rows (`Engine.build_goal_rows` / `reset_rows`, kernels `k_goal_rows` /
`k_reset_rows`), on top of the float64 oracle stand-in of tests/oracle_engine.py.
TEST INFRASTRUCTURE: a goal row is what rebuilds the episode start: (model slot, rand_vec, observability, rand_vec_pass1).
Of the 768 bytes the host reads only the words k_reset_rows checks, the observation and _target_pos, to know which envs
restarted; the stand-in writes them finite for a finite goal and NaN otherwise, as the kernel's rows are.  `reset_rows`
restarts the env from the row's goal by the oracle's reset() with the two passes' vectors, records snapshot id -1 and
skips a row with a non-finite goal, as k_reset_rows leaves such an env unchanged."""
import numpy as np
import torch

from metaworld_b200.engine import ENVSTATE_DTYPE, SNAPSHOT_DTYPE
from oracle_engine import OracleEngine

_OBS = SNAPSHOT_DTYPE.fields["obs"][1] // 4
_TARGET = ENVSTATE_DTYPE.fields["target"][1] // 4


class GoalOracleEngine(OracleEngine):
    def set_envs(self, env_model):
        super().set_envs(env_model)
        self.rows = {}                  # goal rows by rows buffer: {env: (slot, rand_vec, partially_observable, pass 1)}

    def build_goal_rows(self, mask, rand_vec, rand_vec_pass1, partial, rows):
        defs = self.rows.setdefault(rows.data_ptr(), {})
        f = rows.view(torch.float32)
        for e in np.nonzero(mask.numpy())[0]:
            rv = rand_vec[e].numpy().copy()
            rv1 = rv if rand_vec_pass1 is None else rand_vec_pass1[e].numpy().copy()
            defs[e] = (int(self.env_model[e]), rv, bool(partial[e]), rv1)
            ok = np.isfinite(rv).all() and np.isfinite(rv1).all()
            f[e, _OBS:_OBS + 39] = 0.0 if ok else float("nan")
            f[e, _TARGET:_TARGET + 3] = 0.0

    def reset_rows(self, mask, rows, obs):
        defs = self.rows[rows.data_ptr()]
        f = rows.view(torch.float32)
        for e in np.nonzero(mask.numpy())[0]:
            if not torch.isfinite(f[e, _OBS:_OBS + 39]).all():
                continue
            self.snaps.append(defs[e])          # a table entry for the length of the restart only
            try:
                o = self._start(e, len(self.snaps) - 1)
            finally:
                self.snaps.pop()
            self.snap[e] = -1
            obs[e, :39] = torch.from_numpy(o.astype(np.float32))


def goal_vec_env(kind, name, **kw):
    """`oracle_engine.oracle_vec_env` on a `GoalOracleEngine`."""
    from metaworld_b200 import benchmarks as B
    from metaworld_b200 import vector_env as V
    names = {"MT10": B.MT10, "ML10": B.ML10["train"] * 2}.get(name, [name])
    eng = GoalOracleEngine(list(dict.fromkeys(names)))
    return (V.make_mt_envs if kind == "mt" else V.make_ml_envs)(name, engine=eng, **kw)
