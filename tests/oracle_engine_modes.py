"""CPU stand-in for the engine's autoreset modes: `OracleEngine` (tests/oracle_engine.py, SAME_STEP) extended with what
`mw_set_autoreset_mode` / `mw_reset_masked` add to `k_step` / `k_reset_masked` (csrc/mw_engine.cu) per environment, so
that the host code of NEXT_STEP / DISABLED / `reset_mask` can be compared with the reference's stack
(tests/test_autoreset_modes.py).  TEST INFRASTRUCTURE; under SAME_STEP it is `OracleEngine` unchanged."""
import numpy as np
import torch

from metaworld_b200.engine import INFO_KEYS
from oracle_engine import OracleEngine


class OracleEngineModes(OracleEngine):
    def __init__(self, names):
        super().__init__(names)
        self.mode = "SameStep"

    def set_autoreset_mode(self, mode):
        assert mode in ("SameStep", "NextStep", "Disabled")
        self.mode = mode

    def set_envs(self, env_model):
        super().set_envs(env_model)
        self.ended = np.zeros(self.n_envs, dtype=bool)      # MwEnvState.ended

    def _start(self, e, sid):
        self.ended[e] = False
        return super()._start(e, sid)

    def reset_masked(self, mask, obs, snapshot_ids=None):
        for e in np.nonzero(mask.numpy())[0]:
            obs[e, :39] = torch.from_numpy(self._start(e, int(snapshot_ids[e])).astype(np.float32))

    def step(self, actions, obs, reward, term, trunc, info, final_obs, final_info, next_snapshot):
        if self.mode == "SameStep":
            return super().step(actions, obs, reward, term, trunc, info, final_obs, final_info, next_snapshot)
        a = actions.numpy()
        for e, env in enumerate(self.envs):
            if self.ended[e]:          # DISABLED leaves the env and its output rows alone, NEXT_STEP restarts it
                if self.mode == "Disabled":
                    continue
                info[e] = 0; reward[e] = 0.0; term[e] = 0; trunc[e] = 0
                obs[e, :39] = torch.from_numpy(self._start(e, int(next_snapshot[e])).astype(np.float32))
                continue
            o, r, _, _, inf = env.step(a[e])
            self.plen[e] += 1
            self.ret[e] += np.float32(r)
            tr = self.plen[e] >= self.max_steps
            te = self.tos and inf["success"] == 1.0
            info[e, :7] = torch.tensor([float(inf[k]) for k in INFO_KEYS], dtype=torch.float32)
            if info.shape[1] >= 9:
                info[e, 7] = float(r); info[e, 8] = float(int(te) + 2 * int(tr))
            reward[e] = float(r); term[e] = int(te); trunc[e] = int(tr)
            if te or tr:               # the terminal observation stays in obs; the episode return goes to final_info[7]
                final_info[e, 7] = float(self.ret[e])
                self.ended[e] = True
            obs[e, :39] = torch.from_numpy(o.astype(np.float32))

    def get_state(self):
        st = super().get_state()
        st["ended"] = self.ended
        return st
