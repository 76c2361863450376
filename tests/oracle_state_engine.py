"""`OracleEngine` (tests/oracle_engine.py) with the three state calls of `metaworld_b200.engine.Engine`, so that the
host code of `set_state` / `get_env_state` / `_get_obs` can be compared with the reference's own stack without a GPU
(tests/test_set_state.py).
TEST INFRASTRUCTURE: mirrors what `k_set_physics` / `k_get_physics` / `k_observe` do per environment
(csrc/mw_engine.cu): the state is written without a forward pass, qvel passes through the record's float32, and the
observation runs the forward pass (kinematics) before `_get_obs`."""
import numpy as np
import torch

from oracle import mjphys as P
from oracle_engine import OracleEngine


class OracleStateEngine(OracleEngine):
    def set_physics(self, mask, qpos, qvel):
        for e in np.nonzero(mask.numpy())[0]:
            d = self.envs[e].data
            nq, nv = len(d.qpos), len(d.qvel)
            d.qpos = qpos[e, :nq].numpy().copy()
            d.qvel = qvel[e, :nv].numpy().astype(np.float32).astype(np.float64)

    def get_physics(self, qpos, qvel):
        qpos.zero_(); qvel.zero_()
        for e, env in enumerate(self.envs):
            d = env.data
            qpos[e, :len(d.qpos)] = torch.from_numpy(np.array(d.qpos, dtype=np.float64))
            qvel[e, :len(d.qvel)] = torch.from_numpy(np.asarray(d.qvel).astype(np.float32).astype(np.float64))

    def observe(self, mask, obs):
        for e in np.nonzero(mask.numpy())[0]:
            env = self.envs[e]
            P.mj_forward(env.model, env.data)
            obs[e, :39] = torch.from_numpy(env._get_obs().astype(np.float32))


def oracle_vec_env(kind, name, **kw):
    """`make_mt_envs` (kind "mt") or `make_ml_envs` (kind "ml") of `name` on an `OracleStateEngine`."""
    from metaworld_b200 import benchmarks as B
    from metaworld_b200 import vector_env as V
    names = {"MT10": B.MT10, "ML10": B.ML10["train"] * 2}.get(name, [name])
    eng = OracleStateEngine(list(dict.fromkeys(names)))
    return (V.make_mt_envs if kind == "mt" else V.make_ml_envs)(name, engine=eng, **kw)
