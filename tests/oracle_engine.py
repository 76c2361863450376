"""CPU stand-in for `metaworld_b200.engine.Engine` backed by the float64 oracle (oracle/tasks.py): lets the REAL
`MetaWorldVecEnv` host code run without a GPU so that its task streams, autoreset bookkeeping, info layout, episode
statistics and checkpoints can be compared with the reference's own `gym.make_vec(...)` stack in every autoreset mode
(tests/test_refpin_vector.py, tests/test_autoreset_modes.py).
TEST INFRASTRUCTURE: mirrors what `k_step` / `k_reset` / `k_reset_masked` do per environment (csrc/mw_engine.cu), nothing more."""
import numpy as np
import torch

from metaworld_b200.engine import ENVSTATE_DTYPE, INFO_KEYS
from oracle.tasks import TASKS as OT


class OracleEngine:
    def __init__(self, names):
        self.torch = torch
        self.device = torch.device("cpu")
        self.names = list(names)
        self.snaps = []           # (slot, rand_vec, partially_observable)
        self.max_steps, self.tos = 500, False
        self.mode = "SameStep"

    def build_snapshots(self, mi, rvs, po, precise=None, rand_vec_pass1=None):
        first = len(self.snaps)
        for k, (m, rv, p) in enumerate(zip(mi, rvs, po)):
            self.snaps.append((int(m), np.asarray(rv, dtype=np.float64), bool(p), None if rand_vec_pass1 is None else np.asarray(rand_vec_pass1[k], dtype=np.float64)))
        return np.arange(first, len(self.snaps), dtype=np.int32)

    def set_envs(self, env_model):
        self.n_envs = len(env_model)
        self.env_model = np.asarray(env_model, dtype=np.int32)
        self.envs = [OT[self.names[m]]() for m in env_model]
        self.snap = np.zeros(self.n_envs, dtype=np.int64)
        self.plen = np.zeros(self.n_envs, dtype=np.int64)
        self.ret = np.zeros(self.n_envs)
        self.ended = np.zeros(self.n_envs, dtype=bool)      # MwEnvState.ended

    def set_options(self, max_steps, tos, seed):
        self.max_steps, self.tos = int(max_steps), bool(tos)

    def set_autoreset_mode(self, mode):
        assert mode in ("SameStep", "NextStep", "Disabled")
        self.mode = mode

    def set_goal_sets(self, first, count):
        raise NotImplementedError("the device sampler has no CPU stand-in")

    def _start(self, e, sid):
        slot, rv, po, rv1 = self.snaps[sid]
        assert slot == self.env_model[e]
        env = self.envs[e]
        lo, _ = env.random_reset_space()
        env.set_task_vec(rv[: len(lo)], po)
        if rv1 is not None:          # unfrozen rand_vec: pass 1 of reset() used another draw
            seq = [rv1[: len(lo)], rv[: len(lo)]]
            env._get_state_rand_vec = lambda: seq.pop(0) if len(seq) > 1 else seq[0]
        o, _ = env.reset()
        if rv1 is not None:
            del env._get_state_rand_vec
        self.snap[e], self.plen[e], self.ret[e], self.ended[e] = sid, 0, 0.0, False
        return o

    def reset(self, snapshot_ids, obs, env_ids=None):
        ids = range(self.n_envs) if env_ids is None else [int(i) for i in env_ids]
        for k, e in enumerate(ids):
            obs[e, :39] = torch.from_numpy(self._start(e, int(snapshot_ids[k])).astype(np.float32))

    def reset_masked(self, mask, obs, snapshot_ids=None):
        for e in np.nonzero(mask.numpy())[0]:
            obs[e, :39] = torch.from_numpy(self._start(e, int(snapshot_ids[e])).astype(np.float32))

    def step(self, actions, obs, reward, term, trunc, info, final_obs, final_info, next_snapshot):
        a = actions.numpy()
        for e, env in enumerate(self.envs):
            if self.ended[e]:          # NEXT_STEP / DISABLED, the call after the terminal step
                if self.mode == "Disabled":
                    continue           # state and output rows stay as they are
                info[e] = 0; reward[e] = 0.0; term[e] = 0; trunc[e] = 0
                obs[e, :39] = torch.from_numpy(self._start(e, int(next_snapshot[e])).astype(np.float32))
                continue
            o, r, _, _, inf = env.step(a[e])
            self.plen[e] += 1
            self.ret[e] += np.float32(r)
            tr = self.plen[e] >= self.max_steps
            te = self.tos and inf["success"] == 1.0
            row = [float(inf[k]) for k in INFO_KEYS]
            info[e, :7] = torch.tensor(row, dtype=torch.float32)
            if info.shape[1] >= 9:
                info[e, 7] = float(r); info[e, 8] = float(int(te) + 2 * int(tr))
            reward[e] = float(r); term[e] = int(te); trunc[e] = int(tr)
            if (te or tr) and self.mode != "SameStep":     # the terminal observation stays in obs, the env restarts later
                final_info[e, 7] = float(self.ret[e])
                self.ended[e] = True
            elif te or tr:             # SAME_STEP autoreset
                final_obs[e, :39] = torch.from_numpy(o.astype(np.float32))
                final_info[e, :7] = info[e, :7]; final_info[e, 7] = float(self.ret[e])
                o = self._start(e, int(next_snapshot[e]))
            obs[e, :39] = torch.from_numpy(o.astype(np.float32))

    def evaluate(self, actions, obs, out):
        for e, env in enumerate(self.envs):
            r, inf = env.evaluate_state(obs[e, :39].numpy().astype(np.float64), actions[e].numpy())
            out[e, :7] = torch.tensor([float(inf[k]) for k in INFO_KEYS]); out[e, 7] = float(r)

    def get_state(self):
        st = np.zeros(self.n_envs, dtype=ENVSTATE_DTYPE)
        for e, env in enumerate(self.envs):
            st[e]["qpos"][: len(env.data.qpos)] = env.data.qpos
            st[e]["qvel"][: len(env.data.qvel)] = env.data.qvel
            st[e]["snapshot"], st[e]["path_len"], st[e]["ep_return"] = self.snap[e], self.plen[e], self.ret[e]
            st[e]["target"] = np.asarray(env._target_pos, dtype=np.float32)
            if env.obj_init_pos is not None:
                st[e]["obj_init"] = np.asarray(env.obj_init_pos, dtype=np.float32)[:3]
        st["ended"] = self.ended
        return st

    def set_state(self, st):
        raise NotImplementedError("mid-episode physics restore is tested on the device (tests/test_gpu.py)")

    def close(self):
        pass


def oracle_vec_env(kind, name, **kw):
    """`make_mt_envs` (kind "mt") or `make_ml_envs` (kind "ml") of `name` on an `OracleEngine`."""
    from metaworld_b200 import benchmarks as B
    from metaworld_b200 import vector_env as V
    names = {"MT10": B.MT10, "ML10": B.ML10["train"] * 2}.get(name, [name])
    eng = OracleEngine(list(dict.fromkeys(names)))
    return (V.make_mt_envs if kind == "mt" else V.make_ml_envs)(name, engine=eng, **kw)
