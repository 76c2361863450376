"""CPU stand-in for `metaworld_b200.engine.Engine` backed by the float64 oracle (oracle/tasks.py): lets the REAL host
code of `MetaWorldVecEnv`, `SawyerXYZEnvB200` and `metaworld_b200.getters` run without a GPU, so that task streams,
autoreset bookkeeping, info layout, episode statistics, checkpoints, physics state and the state getters can be compared
with the reference's own stack (tests/test_refpin_vector.py, tests/test_autoreset_modes.py, tests/test_set_state.py,
tests/test_query.py, tests/test_query_refstack.py).
TEST INFRASTRUCTURE: each call mirrors what its kernel (csrc/mw_engine.cu) does per environment, nothing more:
* `reset` / `reset_masked` / `step` mirror `k_reset` / `k_reset_masked` / `k_step`;
* `set_physics` mirrors `k_set_physics`: the state is written without a forward pass, qvel through the record's float32;
* `get_physics` mirrors `k_get_physics`: qvel as the record's float32 holds it;
* `observe` mirrors `k_observe`: the forward pass (kinematics) of the current state, then `_get_obs`;
* `query` mirrors `k_query`: a forward pass of the current state, then the observation frame without committing the
  frame stack, the named poses (NaN for a missing name) and touching_object of the slot's geom.  Sites a task's
  reset_model places through model.site(name).pos are posed as the kernel poses them (their body + _target_pos /
  obj_init_pos): the oracle leaves some of them at the model file's place;
* `build_goal_rows` / `reset_rows` mirror `k_goal_rows` / `k_reset_rows`.  A goal row is what rebuilds the episode
  start: (model slot, rand_vec, observability, rand_vec_pass1).  Of the 768 bytes the host reads only the words
  k_reset_rows checks, the observation and _target_pos, to know which envs restarted; the stand-in writes them finite
  for a finite goal and NaN otherwise, as the kernel's rows are.  `reset_rows` restarts the env from the row's goal by
  the oracle's reset() with the two passes' vectors, records snapshot id -1 and skips a row with a non-finite goal, as
  k_reset_rows leaves such an env unchanged;
* `save_states` / `load_states` mirror `k_save_states` / `k_load_states`.  An oracle env's state lives in C memory that
  cannot be copied, so a saved row is what rebuilds it: the definition of the episode's start (a snapshot's or a goal
  row's), the calls that changed the env since (steps, set_physics, observe) and the counters.  Loading restarts the
  target env from that definition and replays the calls, so the target continues exactly as the source would.  The
  record rows get the state record (the host reads the ended mark there) and the model slot; a row out of range or of
  another model is skipped, as k_load_states leaves such an env unchanged."""
import numpy as np
import torch
from scipy.spatial.transform import Rotation

from metaworld_b200 import modelzoo
from metaworld_b200.engine import ENVSTATE_DTYPE, INFO_KEYS, SNAPSHOT_DTYPE
from metaworld_b200.tasks import MOVED_SITES, TASKS
from oracle import mjphys as P
from oracle.tasks import TASKS as OT

_OBS = SNAPSHOT_DTYPE.fields["obs"][1] // 4
_TARGET = ENVSTATE_DTYPE.fields["target"][1] // 4


class OracleEngine:
    def __init__(self, names):
        self.torch = torch
        self.device = torch.device("cpu")
        self.names = list(names)
        self.snaps = []           # episode starts: (slot, rand_vec, partially_observable, rand_vec_pass1)
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
        self.start = [None] * self.n_envs                   # each env's episode start, in the form of a snaps entry
        self.log = [[] for _ in range(self.n_envs)]         # what changed each env since its episode start
        self.saved = {}                                     # save_states rows, by records buffer
        self.rows = {}                                      # goal rows, by rows buffer

    def set_options(self, max_steps, tos, seed):
        self.max_steps, self.tos = int(max_steps), bool(tos)

    def set_autoreset_mode(self, mode):
        assert mode in ("SameStep", "NextStep", "Disabled")
        self.mode = mode

    def set_goal_sets(self, first, count):
        raise NotImplementedError("the device sampler has no CPU stand-in")

    def _start(self, e, sid, start=None):
        """Restarts env e from `start` (default: snapshot `sid`) and records `sid` as its snapshot id."""
        start = self.snaps[sid] if start is None else start
        slot, rv, po, rv1 = start
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
        self.start[e], self.log[e] = start, []
        return o

    def reset(self, snapshot_ids, obs, env_ids=None):
        ids = range(self.n_envs) if env_ids is None else [int(i) for i in env_ids]
        for k, e in enumerate(ids):
            obs[e, :39] = torch.from_numpy(self._start(e, int(snapshot_ids[k])).astype(np.float32))

    def reset_masked(self, mask, obs, snapshot_ids=None):
        for e in np.nonzero(mask.numpy())[0]:
            obs[e, :39] = torch.from_numpy(self._start(e, int(snapshot_ids[e])).astype(np.float32))

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
            if torch.isfinite(f[e, _OBS:_OBS + 39]).all():
                obs[e, :39] = torch.from_numpy(self._start(e, -1, defs[e]).astype(np.float32))

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
            self.log[e].append(("step", a[e].copy()))
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
            if getattr(env, "init_tcp", None) is not None:
                st[e]["init_tcp"] = np.asarray(env.init_tcp, dtype=np.float32)
        st["ended"] = self.ended
        return st

    def set_state(self, st):
        raise NotImplementedError("mid-episode physics restore is tested on the device (tests/test_gpu.py)")

    def save_states(self, records, record_model, hints, mask=None):
        st = self.get_state()
        saved = self.saved.setdefault(records.data_ptr(), {})
        for e in range(self.n_envs) if mask is None else np.nonzero(mask.numpy())[0]:
            records[e] = torch.from_numpy(np.frombuffer(st[e].tobytes(), dtype=np.uint8).copy())
            record_model[e] = int(self.env_model[e])
            saved[e] = (self.start[e], int(self.snap[e]), list(self.log[e]), int(self.plen[e]), float(self.ret[e]),
                        bool(self.ended[e]))

    def load_states(self, records, record_model, hints, mask=None, src=None):
        saved = self.saved[records.data_ptr()]
        for e in range(self.n_envs) if mask is None else np.nonzero(mask.numpy())[0]:
            s = e if src is None else int(src[e])
            if not (0 <= s < records.shape[0] and int(record_model[s]) == self.env_model[e]):
                continue
            start, sid, log, plen, ret, ended = saved[s]
            self._start(e, sid, start)
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

    def set_physics(self, mask, qpos, qvel):
        for e in np.nonzero(mask.numpy())[0]:
            d = self.envs[e].data
            nq, nv = len(d.qpos), len(d.qvel)
            d.qpos = qpos[e, :nq].numpy().copy()
            d.qvel = qvel[e, :nv].numpy().astype(np.float32).astype(np.float64)
            self.log[e].append(("set", np.array(d.qpos, dtype=np.float64), np.array(d.qvel, dtype=np.float64)))

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
            self.log[e].append(("observe",))

    def query(self, mask, frame=None, pose=None, frames=None, touching=None, main_geom=None):
        for e in np.nonzero(mask.numpy())[0]:
            env = self.envs[e]
            task = self.names[self.env_model[e]]
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
                move = MOVED_SITES.get(task, {}).get(name) if kind == "site" else None
                if move is not None:            # reset_model set model.site(name).pos: parent body + the env's vector
                    m = modelzoo.full_model(TASKS[task].xml)
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

    def close(self):
        pass


def oracle_vec_env(kind, name, **kw):
    """`make_mt_envs` (kind "mt") or `make_ml_envs` (kind "ml") of `name` on an `OracleEngine`."""
    from metaworld_b200 import benchmarks as B
    from metaworld_b200 import vector_env as V
    names = {"MT10": B.MT10, "ML10": B.ML10["train"] * 2}.get(name, [name])
    eng = OracleEngine(list(dict.fromkeys(names)))
    return (V.make_mt_envs if kind == "mt" else V.make_ml_envs)(name, engine=eng, **kw)
