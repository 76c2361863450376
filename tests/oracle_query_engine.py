"""`OracleStateEngine` (tests/oracle_state_engine.py) with `Engine.query`, so that the host code of `query_torch` and of the
reference's getters (call / get_attr, the bare env) runs without a GPU.
TEST INFRASTRUCTURE: mirrors what `k_query` does per environment (csrc/mw_engine.cu): a forward pass of the current
state, then the observation frame without committing the frame stack, the named poses (NaN for a missing name) and
touching_object of the slot's geom.  Sites a task's reset_model places through model.site(name).pos are posed as the
kernel poses them (their body + _target_pos / obj_init_pos): the oracle leaves some of them at the model file's place."""
import numpy as np
import torch
from scipy.spatial.transform import Rotation

from metaworld_b200 import modelzoo
from metaworld_b200.tasks import MOVED_SITES, TASKS
from oracle import mjphys as P
from oracle_state_engine import OracleStateEngine


class OracleQueryEngine(OracleStateEngine):
    def get_state(self):
        st = super().get_state()
        for e, env in enumerate(self.envs):            # the record keeps init_tcp (k_snapshot)
            if getattr(env, "init_tcp", None) is not None:
                st[e]["init_tcp"] = np.asarray(env.init_tcp, dtype=np.float32)
        return st

    def query(self, mask, frame=None, pose=None, frames=None, touching=None, main_geom=None):
        for e in np.nonzero(mask.numpy())[0]:
            env = self.envs[e]
            P.mj_forward(env.model, env.data)
            if frame is not None:
                frame[e] = torch.from_numpy(np.asarray(env._get_curr_obs_combined_no_goal(), dtype=np.float32))
            for k, (kind, name) in enumerate(frames or ()):
                try:
                    v = getattr(env.data, kind)(name)
                except (KeyError, ValueError):   # the oracle's name lookup
                    pose[e, k] = float("nan")
                    continue
                xyzw = Rotation.from_matrix(np.asarray(v.xmat, dtype=np.float64).reshape(3, 3)).as_quat()
                xpos = np.asarray(v.xpos, dtype=np.float64)
                move = MOVED_SITES.get(self.names[self.env_model[e]], {}).get(name) if kind == "site" else None
                if move is not None:            # reset_model set model.site(name).pos: parent body + the env's vector
                    m = modelzoo.full_model(TASKS[self.names[self.env_model[e]]].xml)
                    body = m.names["body"][m.arrays["site_bodyid"][m.names["site"].index(name)]]
                    vec = env._target_pos if move == "target" else np.asarray(env.obj_init_pos) + np.asarray(move[1])
                    xpos = np.asarray(env.data.body(body).xpos, dtype=np.float64) + np.asarray(vec, dtype=np.float64)
                pose[e, k, :3] = torch.from_numpy(xpos)
                pose[e, k, 3:] = torch.from_numpy(np.r_[xyzw[3], xyzw[:3]])
            if touching is not None:
                g = main_geom[self.env_model[e]]
                try:
                    touching[e] = bool(g is not None and env.touching_object(env.data.geom(g).id))
                except (KeyError, ValueError):   # no such geom in this model: collider -1
                    touching[e] = False
