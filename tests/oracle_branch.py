"""CPU stand-in for the engine's saved states (`Engine.save_states` / `load_states`, kernels `k_save_states` /
`k_load_states`), on top of the float64 oracle stand-in of tests/oracle_engine.py.
TEST INFRASTRUCTURE: an oracle env's state lives in C memory that cannot be copied, so a saved row is what rebuilds it:
the episode's snapshot id, the calls that changed the env since (steps, set_physics, observe) and the counters.  Loading
restarts the target env from that snapshot and replays the calls, so the target continues exactly as the source would.
The record rows get the state record (the host reads the ended mark there) and the model slot; a row out of range or of
another model is skipped, as k_load_states leaves such an env unchanged."""
import numpy as np
import torch

from oracle import mjphys as P
from oracle_engine import OracleEngine


class BranchOracleEngine(OracleEngine):
    def set_envs(self, env_model):
        super().set_envs(env_model)
        self.log = [[] for _ in range(self.n_envs)]     # what changed each env since its episode's snapshot
        self.fresh = np.zeros(self.n_envs, dtype=bool)  # restarted during the current call
        self.saved = {}                                 # save_states rows, by records buffer

    def _start(self, e, sid):
        o = super()._start(e, sid)
        self.log[e], self.fresh[e] = [], True
        return o

    def step(self, actions, *args):
        was_ended = self.ended.copy()
        self.fresh[:] = False
        super().step(actions, *args)
        a = actions.numpy()
        for e in np.nonzero(~was_ended & ~self.fresh)[0]:     # stepped and not restarted by a SAME_STEP autoreset
            self.log[e].append(("step", a[e].copy()))

    def set_physics(self, mask, qpos, qvel):
        super().set_physics(mask, qpos, qvel)
        for e in np.nonzero(mask.numpy())[0]:
            d = self.envs[e].data
            self.log[e].append(("set", np.array(d.qpos, dtype=np.float64), np.array(d.qvel, dtype=np.float64)))

    def observe(self, mask, obs):
        super().observe(mask, obs)
        for e in np.nonzero(mask.numpy())[0]:
            self.log[e].append(("observe",))

    def save_states(self, records, record_model, hints, mask=None):
        st = self.get_state()
        saved = self.saved.setdefault(records.data_ptr(), {})
        for e in range(self.n_envs) if mask is None else np.nonzero(mask.numpy())[0]:
            records[e] = torch.from_numpy(np.frombuffer(st[e].tobytes(), dtype=np.uint8).copy())
            record_model[e] = int(self.env_model[e])
            saved[e] = (int(self.snap[e]), list(self.log[e]), int(self.plen[e]), float(self.ret[e]), bool(self.ended[e]))

    def load_states(self, records, record_model, hints, mask=None, src=None):
        saved = self.saved[records.data_ptr()]
        for e in range(self.n_envs) if mask is None else np.nonzero(mask.numpy())[0]:
            s = e if src is None else int(src[e])
            if not (0 <= s < records.shape[0] and int(record_model[s]) == self.env_model[e]):
                continue
            sid, log, plen, ret, ended = saved[s]
            self._start(e, sid)
            env = self.envs[e]
            for op in log:
                if op[0] == "step":
                    env.step(op[1])
                elif op[0] == "set":
                    env.data.qpos, env.data.qvel = op[1].copy(), op[2].copy()
                else:
                    P.mj_forward(env.model, env.data)
                    env._get_obs()
            self.log[e] = list(log)
            self.plen[e], self.ret[e], self.ended[e] = plen, ret, ended


def branch_vec_env(kind, name, **kw):
    """`oracle_engine.oracle_vec_env` on a `BranchOracleEngine`."""
    from metaworld_b200 import benchmarks as B
    from metaworld_b200 import vector_env as V
    names = {"MT10": B.MT10, "ML10": B.ML10["train"] * 2}.get(name, [name])
    eng = BranchOracleEngine(list(dict.fromkeys(names)))
    return (V.make_mt_envs if kind == "mt" else V.make_ml_envs)(name, engine=eng, **kw)
