"""Drop-in vector environment over the CUDA engine.

Stands where the reference puts ``gymnasium.vector.SyncVectorEnv([...partial(_init_each_env ...)])``
(metaworld/__init__.py:460-604): same construction kwargs, same ``reset`` / ``step`` return shapes and dtypes,
SAME_STEP autoreset with ``final_obs`` / ``final_info`` (``autoreset_mode`` selects gymnasium's NEXT_STEP or DISABLED
instead; ``reset(options={"reset_mask": m})`` resets some envs), the per-env wrapper stack folded in
(TimeLimit, AutoTerminateOnSuccessWrapper, OneHotWrapper, RecordEpisodeStatistics,
Random/PseudoRandomTaskSelectWrapper, CheckpointWrapper -- metaworld/wrappers.py) and the ``call`` / ``get_attr`` /
``set_attr`` names that ``metaworld/evaluation.py`` and the reference tests use.

Extension over the reference: ``num_envs`` may be any multiple of the number of env types (the reference
ignores it); env ``e`` has type ``e % n_types`` (task ids interleaved) and replica ``e // n_types``.  Replica
``r`` seeds its task-selection RNG with ``seed + r`` so replica 0 reproduces the reference stream.

The numpy API (`reset`, `step`) moves actions host->device and results device->host every call; the
``*_torch`` variants keep everything on the GPU and never synchronise.

Task selection on autoreset.  The reference draws the next task inside ``reset`` (wrappers.py:116-119), i.e. after the
terminal step.  The kernel needs the snapshot id of the next episode BEFORE the step that may end the episode, so the
host draws one task ahead ("pending").  The draw is speculative: whenever the sampler state becomes observable
(checkpoint, ``toggle_sample_tasks_on_reset``, ``sample_tasks``, an explicit ``reset``) it is either consumed as the
draw the reference would make at that point or rewound, so the task sequence and the RNG stream are the reference's.
"""
from __future__ import annotations

import base64
from typing import Any, NamedTuple

import numpy as np

from . import _gym
from .benchmarks import Task, draw_rand_vec, make_task, reference_env_id
from .engine import ENVSTATE_DTYPE, INFO_KEYS, MAXDOF, MAXNQ, NCONV, SNAPSHOT_DTYPE, Engine, expert_actions
from .getters import STATE_ATTRS, STATE_CALLS, StateGetters, _quat2mat  # noqa: F401  (_quat2mat: still importable from here)
from .tasks import TASK_IDS, TASKS

MAX_PATH_LENGTH = 500     # SawyerXYZEnv.max_path_length (sawyer_xyz_env.py:152): truncates whatever TimeLimit says


def _serialize_task(task: Task) -> dict:          # metaworld/wrappers.py:35-39
    return {"env_name": task.env_name, "data": base64.b64encode(task.data).decode("ascii")}


def _deserialize_task(d: dict) -> Task:            # metaworld/wrappers.py:42-47
    assert "env_name" in d and "data" in d
    return Task(env_name=d["env_name"], data=base64.b64decode(d["data"]))


_AUTORESET_MODES = {"SameStep": "same_step", "NextStep": "next_step", "Disabled": "disabled"}


def parse_autoreset_mode(mode):
    """gymnasium.vector.AutoresetMode member or its value ("SameStep", "NextStep", "Disabled"; None = SAME_STEP) ->
    that value; anything else raises ValueError."""
    if mode is None:
        return "SameStep"
    v = getattr(mode, "value", mode)
    if type(mode).__name__ == "AutoresetMode" and v in _AUTORESET_MODES or isinstance(mode, str) and mode in _AUTORESET_MODES:
        return v
    raise ValueError(f"autoreset_mode must be a gymnasium.vector.AutoresetMode or one of {sorted(_AUTORESET_MODES)}, got {mode!r}")


def _rng(seed):
    return np.random.Generator(np.random.PCG64(seed)) if seed is not None else np.random.default_rng()


class _SubEnv:
    """Host mirror of one sub-env's wrapper state (task list, RNGs, flags)."""

    def __init__(self, name, tasks, seed, pseudorandom, env_id):
        self.task_name = name
        self.env_id = env_id
        self.tasks = list(tasks)
        # env.seed(seed) (metaworld/__init__.py:428, sawyer_xyz_env.py:274-292) seeds env.np_random -- which the
        # task-select wrappers use (Wrapper.np_random is the wrapped env's) -- and the three spaces with the same seed
        self.np_random = _rng(seed)
        self.space_rng = {k: _rng(seed) for k in ("action_space", "obs_space", "goal_space")}
        self.pseudorandom = pseudorandom
        self.sample_tasks_on_reset = not pseudorandom
        self.current_task_idx = -1
        self.current_task: Task | None = None
        self.pending: Task | None = None
        self._pre = None          # sampler state before the speculative draw of `pending`

    def next_task(self):
        if self.pseudorandom:     # PseudoRandomTaskSelectWrapper._set_pseudo_random_task (wrappers.py:156-160)
            self.current_task_idx = (self.current_task_idx + 1) % len(self.tasks)
            if self.current_task_idx == 0:
                self.np_random.shuffle(self.tasks)
            return self.tasks[self.current_task_idx]
        idx = self.np_random.choice(len(self.tasks))   # RandomTaskSelectWrapper._set_random_task (wrappers.py:98-100)
        return self.tasks[idx]

    def draw_pending(self):
        """Task of the next episode, drawn one episode early (see module docstring)."""
        if self.sample_tasks_on_reset:
            self._pre = (list(self.tasks), self.current_task_idx, self.np_random.bit_generator.state)
            self.pending = self.next_task()
        else:
            self._pre = None
            self.pending = self.current_task

    def rewind_pending(self):
        if self._pre is not None:
            self.tasks, self.current_task_idx, self.np_random.bit_generator.state = self._pre
        self._pre = None
        self.pending = None

    def take_for_reset(self):
        """What the task-select wrapper's ``reset`` does (wrappers.py:116-119 / 181-184)."""
        if self.sample_tasks_on_reset:
            if self._pre is not None:          # the speculative draw IS the draw the reference makes now
                self.current_task, self._pre, self.pending = self.pending, None, None
            else:
                self.current_task = self.next_task()
        elif self.current_task is None:
            self.current_task = self.next_task()


class _Mirrored:
    """One per-env value that the numpy calls read and write on the host (a numpy array) and the `_torch` calls on the
    device (a tensor).  A write records the side it happened on and drops the other copy; a read of the other side
    converts once (`to_host` / `to_device`) and keeps both copies until the next write."""

    def __init__(self, to_host, to_device, host=None):
        self._to_host, self._to_device = to_host, to_device
        self._host, self._device = host, None

    def set(self, host=None, device=None):
        """The value was just written: on the host, on the device, or on both when the two are equal."""
        self._host, self._device = host, device

    def on_host(self):
        return self._host is not None

    def host(self, write=False):
        """The host copy; `write`: the caller changes it in place, so the device copy is dropped."""
        if self._host is None:
            self._host = self._to_host(self._device)
        if write:
            self._device = None
        return self._host

    def device(self, write=False):
        """The device copy; `write`: the caller changes it in place, so the host copy is dropped."""
        if self._device is None:
            self._device = self._to_device(self._host)
        if write:
            self._host = None
        return self._device


_ENDED_WORD = ENVSTATE_DTYPE.fields["ended"][1] // 4      # the ended mark's float32 word in a 512-byte state record
# the float32 words of a 768-byte goal row (engine.build_goal_rows) that mw_reset_rows checks: _target_pos and the observation
_ROW_TARGET = ENVSTATE_DTYPE.fields["target"][1] // 4
_ROW_OBS = SNAPSHOT_DTYPE.fields["obs"][1] // 4


class EnvStates:
    """Every env's complete state as `MetaWorldVecEnv.save_states` saved it, on the device; only the env that saved it can
    load it (`load_states`, `load_states_torch`).  Row e is env e's state at the save; a row that was not selected then
    holds no state (model id -1), and loading it fails like a model mismatch.
    * `records` uint8 [N, 512], `model` int32 [N], `hints` float32 [N, NCONV, 4]: the engine's state records (the ended
      mark of NEXT_STEP / DISABLED included), model slots and separating-axis hints;
    * `raw`: float32 [N, 39], each env's last base observation; `obs`: the last observation returned to the caller
      (a numpy array when the last call was the numpy `reset` / `step`, else a device tensor);
    * `post`: the optional wrappers' per-env rows (`StepPost.save_rows`);
    * `ep_len`, `tasks`: the host mirrors of the episode lengths and the running tasks;
    * `goal`: float64 [N, 6], the running goals of the envs on a `reset_goals` goal (None before the first such reset)."""

    def __init__(self, owner, records, model, hints, raw, obs, post, ep_len, tasks, goal):
        self.owner, self.records, self.model, self.hints = owner, records, model, hints
        self.raw, self.obs, self.post, self.ep_len, self.tasks, self.goal = raw, obs, post, ep_len, tasks, goal

    def ended(self):
        """bool [N] device tensor: the rows saved between a terminal step and its restart."""
        import torch
        return self.records.view(torch.float32)[:, _ENDED_WORD] != 0


class Rollout(NamedTuple):
    """What `MetaWorldVecEnv.rollout_torch` returns for K candidate action sequences of H steps over N envs: device tensors
    (numpy arrays from `rollout`).  Row [k, h, e] is step h of candidate k from env e's current state.
    * `reward` float32 [K, H, N], `info` float32 [K, H, N, 7] (INFO_KEYS order): the base env's raw reward and infos;
    * `terminated`, `truncated` bool [K, H, N]: the step that ends the row's episode;
    * `ended` bool [K, H, N]: the episode ended before this step (reward, info and obs are zero);
    * `obs` float32 [K, H, N, 39] or None: the base observation, the terminal one on the ending step;
    * `faults` int32 [K, N]: fault bits 1 / 2 / 4 / 8 (`Engine.FAULTS`) OR-ed over the row's live steps;
    * `contacts_dropped` int32 [K, N]: the contacts the row's live steps dropped."""
    reward: Any
    info: Any
    terminated: Any
    truncated: Any
    ended: Any
    obs: Any
    faults: Any
    contacts_dropped: Any


class MetaWorldVecEnv(_gym.VectorEnvBase):
    metadata = {"render_modes": [], "autoreset_mode": "same_step"}

    def __init__(self, env_names, tasks_per_env, num_envs=None, seed=None, use_one_hot=False, num_tasks=None,
                 env_ids=None, max_episode_steps=None, terminate_on_success=False, task_select="random",
                 reward_function_version="v2", device=0, engine=None, recurrent_info_in_obs=False,
                 normalize_reward_in_recurrent_info=True, reward_normalization_method=None, reward_alpha=0.001,
                 normalize_observations=False, checkpoint_env_ids=None, type_seeds=None, autoreset_mode=None, **unused):
        if reward_function_version != "v2":
            raise NotImplementedError("only the default v2 rewards are implemented on the device")
        # gymnasium's AutoresetMode (SyncVectorEnv): SameStep (default) / NextStep / Disabled
        self.autoreset_mode = parse_autoreset_mode(autoreset_mode)
        self.metadata = dict(type(self).metadata, autoreset_mode=_AUTORESET_MODES[self.autoreset_mode])
        n_types = len(env_names)
        num_envs = n_types if num_envs is None else int(num_envs)
        if num_envs < n_types:
            raise ValueError(f"num_envs ({num_envs}) must be at least the number of env types ({n_types})")
        self.num_envs = num_envs
        self.n_types = n_types
        self.env_names = list(env_names)
        self.max_episode_steps = int(max_episode_steps or MAX_PATH_LENGTH)
        self.terminate_on_success = bool(terminate_on_success)
        self.use_one_hot = bool(use_one_hot)
        self.num_tasks = int(num_tasks or n_types)
        self.env_ids = list(range(n_types)) if env_ids is None else list(env_ids)
        self._seed = 0 if seed is None else int(seed)
        # one model slot per distinct env name
        uniq = list(dict.fromkeys(env_names))
        self.engine = engine or Engine(uniq, device=device)
        self._own_engine = engine is None
        torch = self.engine.torch
        self.torch = torch
        self.device = self.engine.device
        self._slot = [uniq.index(n) for n in env_names]
        self._slot_of_name = {n: uniq.index(n) for n in uniq}
        # snapshots: one per distinct (model slot, rand_vec, partially_observable)
        self._snap_of: dict = {}
        self._task_of_snap: dict = {}
        self._ensure_snapshots([tk for tasks in tasks_per_env for tk in tasks])
        # CheckpointWrapper ids (metaworld/__init__.py:455: f"{env_cls}_{env_id}"; env_id is None for the ML benchmarks)
        ck_ids = checkpoint_env_ids if checkpoint_env_ids is not None else self.env_ids
        self.sub = []
        for e in range(num_envs):
            t_i, rep = e % n_types, e // n_types
            # every env type shares `seed` (metaworld/__init__.py:497); the custom-mt entry point gives type i seed + i (:762)
            s = (None if seed is None else seed + rep) if type_seeds is None else (None if type_seeds[t_i] is None else type_seeds[t_i] + rep)
            eid = reference_env_id(env_names[t_i], ck_ids[t_i]) if env_names[t_i] in TASKS else f"{env_names[t_i]}_{ck_ids[t_i]}"
            if rep:       # replicas are an extension (the reference has one sub-env per id): keep their ids distinct
                eid += f".r{rep}"
            self.sub.append(_SubEnv(env_names[t_i], tasks_per_env[t_i], s, task_select != "random", eid))
        self._env_model = np.array([self._slot[e % n_types] for e in range(num_envs)], dtype=np.int32)   # env -> model slot
        self.engine.set_envs(self._env_model)
        self._getters = StateGetters(self.engine, [s.task_name for s in self.sub])
        self._set_engine_options()
        if self.autoreset_mode != "SameStep":
            self.engine.set_autoreset_mode(self.autoreset_mode)
        # spaces
        T = self.num_tasks if self.use_one_hot else 0
        self.obs_dim = 39 + T
        self.obs_dtype = np.float32 if self.use_one_hot else np.float64
        inf = np.full(14, np.inf)
        hl, hh = np.array([-0.525, 0.348, -0.0525]), np.array([0.525, 1.025, 0.7])
        # goal bounds are [0, 0]: the reference builds the space at construction, when every env is still partially
        # observable (sawyer_xyz_env.py:208,546-558), and the wrappers keep that Box (wrappers.py:19-30)
        lo = np.hstack((hl, -1.0, -inf, hl, -1.0, -inf, np.zeros(3), np.zeros(T)))
        hi = np.hstack((hh, 1.0, inf, hh, 1.0, inf, np.zeros(3), np.ones(T)))
        self.single_observation_space = _gym.Box(lo.astype(self.obs_dtype), hi.astype(self.obs_dtype), dtype=self.obs_dtype)
        self.single_action_space = _gym.Box(-np.ones(4, np.float32), np.ones(4, np.float32), dtype=np.float32, seed=seed)
        self.observation_space = _gym.batch_space(self.single_observation_space, num_envs)
        self.action_space = _gym.batch_space(self.single_action_space, num_envs, seed=seed)
        # device buffers
        N = num_envs
        dev = self.device
        self.d_obs = torch.zeros(N, self.obs_dim, device=dev)
        if self.use_one_hot:
            ids = torch.tensor([self.env_ids[e % n_types] for e in range(N)], device=dev)
            self.d_obs[torch.arange(N, device=dev), 39 + ids] = 1.0
        self.d_final_obs = self.d_obs.clone()
        self.d_env_obs = self.d_obs.clone()            # observe_torch's output
        self.d_all = torch.ones(N, dtype=torch.bool, device=dev)
        self.d_env_model = torch.from_numpy(self._env_model).to(dev)   # load_states_torch's check
        # reset_goals: each env's observability (constant over its task list) and, allocated on first use, the goal rows,
        # that flag on the device and the running goal of every env whose record has snapshot id -1
        self._partial = np.array([bool(s.tasks[0].unpack()["partially_observable"]) for s in self.sub])
        self._goal_bufs = None
        # the numpy API's outputs: the 39 columns k_step writes, packed (stride 39): the constant one-hot columns never cross
        # the bus, and the host converts a contiguous [N, 39] block
        self.d_obs39 = torch.zeros(N, 39, device=dev)
        # the buffer whose first 39 columns hold every env's base observation as the last reset / step left it (before the
        # optional wrappers): `d_obs` after `reset` and the torch calls, `d_obs39` after the numpy `step`; the default
        # input of `expert_actions_torch`
        self._d_raw = self.d_obs
        self._d_expert_ids = None
        self._rollout_hints = None                     # rollout_torch's hint workspace [K * N, NCONV, 4], grown with K
        self.d_final_obs39 = torch.zeros(N, 39, device=dev)
        self.d_reward = torch.zeros(N, device=dev)
        self.d_term = torch.zeros(N, dtype=torch.uint8, device=dev)
        self.d_trunc = torch.zeros(N, dtype=torch.uint8, device=dev)
        self.d_small = torch.zeros(N, 9, device=dev)        # info[7], reward, flags (terminated + 2 truncated): one D2H record
        self.d_info = self.d_small[:, :7]
        self.d_final_info = torch.zeros(N, 8, device=dev)
        self.d_actions = torch.zeros(N, 4, device=dev)
        self.d_next = torch.zeros(N, dtype=torch.int32, device=dev)
        self.d_cur = torch.zeros(N, dtype=torch.int32, device=dev)
        self.d_idx = torch.zeros(N, dtype=torch.int64, device=dev)
        on_gpu = self.device.type == "cuda"      # (the host-logic tests drive this class with a CPU stand-in for the engine)
        pin = (lambda t: t.pin_memory()) if on_gpu else (lambda t: t)
        self.h_actions = pin(torch.zeros(N, 4))
        self.h_next = pin(torch.zeros(N, dtype=torch.int32))
        self.h_idx = pin(torch.zeros(N, dtype=torch.int64))
        self.h_obs = pin(torch.zeros(N, self.obs_dim))
        self.h_obs39 = pin(torch.zeros(N, 39))
        self.h_final_obs39 = pin(torch.zeros(N, 39))
        self.h_small = pin(torch.zeros(N, 9))
        self.h_final_info = pin(torch.zeros(N, 8))
        self._next_ids = np.zeros(N, dtype=np.int32)
        self._ep_len = np.zeros(N, dtype=np.int64)
        self._closed = False
        self._needs_reset = True
        self._device_sampler = False
        # NEXT_STEP / DISABLED: envs whose last step ended their episode and that have not restarted (the engine's `ended`
        # flag).  Its device copy is always this one buffer, which step_torch writes in place
        d_marks = torch.zeros(N, dtype=torch.bool, device=dev)
        self._autoreset_envs = _Mirrored(lambda d: d.cpu().numpy().copy(), lambda h: d_marks.copy_(torch.from_numpy(h)),
                                         host=np.zeros(N, dtype=bool))
        # what the last call returned (the unmasked rows of a partial reset)
        self._returned_obs = _Mirrored(lambda d: d.cpu().numpy().astype(self.obs_dtype), self._obs_to_device)
        # optional per-sub-env wrappers of the reference that sit above the one-hot wrapper (metaworld/__init__.py:437-444);
        # one instance (one set of statistics) serves both `step` and `step_torch`
        from .post import StepPost
        if recurrent_info_in_obs:
            self.obs_dtype = np.float32
        self.post = StepPost(N, recurrent_info_in_obs, normalize_reward_in_recurrent_info, reward_normalization_method, reward_alpha,
                             normalize_observations, obs_dtype=self.obs_dtype, same_step=self.autoreset_mode == "SameStep")
        if self.post.recurrent or self.post.norm_obs:
            # RNNBasedMetaRLWrapper (obs + action + reward + done, wrappers.py:55-62) and gymnasium.wrappers.NormalizeObservation
            # both declare an unbounded float32 space
            D = self.obs_dim + self.post.extra
            self.single_observation_space = _gym.Box(np.full(D, -np.inf, np.float32), np.full(D, np.inf, np.float32), dtype=np.float32)
            self.observation_space = _gym.batch_space(self.single_observation_space, num_envs)

    # ------------------------------------------------------------------ helpers
    def _set_engine_options(self):
        # SawyerXYZEnv truncates at its own max_path_length = 500 whatever the TimeLimit wrapper says (sawyer_xyz_env.py:634)
        self.engine.set_options(min(self.max_episode_steps, MAX_PATH_LENGTH), self.terminate_on_success, self._seed)

    def _obs_to_device(self, obs):
        """A returned numpy observation as a float32 device tensor.  Without the optional wrappers that tensor is `d_obs`
        itself, so a masked restart writes its rows straight into it."""
        x = self.torch.from_numpy(np.asarray(obs, dtype=np.float32))
        return x.to(self.device) if self.post.active else self.d_obs.copy_(x)

    def _host_mask(self, env_mask, name="env_mask"):
        """A numpy bool mask [num_envs], checked; None = every env."""
        N = self.num_envs
        m = np.ones(N, dtype=bool) if env_mask is None else np.asarray(env_mask)
        if m.shape != (N,) or m.dtype != np.bool_:
            raise ValueError(f"{name} must be a numpy bool array of shape ({N},), got {m.dtype} {m.shape}")
        return m

    def _device_mask(self, env_mask):
        """A numpy bool mask [num_envs], checked and uploaded for a `_torch` call; None (every env) stays None."""
        return None if env_mask is None else self.torch.from_numpy(self._host_mask(env_mask)).to(self.device)

    def _check_tensor(self, name, x, dtype, shape, min_cols=None, contiguous=False):
        """Raises ValueError unless `x` is a tensor on this env's device of `dtype` ("integer": any dtype that is not
        floating point) and of `shape`; with `min_cols`, of shape [*shape, >= min_cols] with unit column stride (a column
        slice of a wider tensor passes); with `contiguous`, contiguous."""
        t = self.torch
        ok = isinstance(x, t.Tensor) and x.device == self.device
        ok = ok and (not x.is_floating_point() if dtype == "integer" else x.dtype == dtype)
        if min_cols is None:
            ok = ok and tuple(x.shape) == shape
            want = str(shape)
        else:
            ok = ok and x.dim() == len(shape) + 1 and tuple(x.shape[:-1]) == shape and x.shape[-1] >= min_cols and x.stride(-1) == 1
            want = f"({', '.join(map(str, shape))}, >= {min_cols})"
        if not (ok and (not contiguous or x.is_contiguous())):
            kind = "integer" if dtype == "integer" else str(dtype).removeprefix("torch.")
            raise ValueError(f"{name} must be a {'contiguous ' if contiguous else ''}{kind} tensor of shape {want} on {self.device}")

    def _torch_mask(self, env_mask, name="env_mask"):
        """A bool device tensor [num_envs], checked and made contiguous; None = every env."""
        if env_mask is None:
            return self.d_all
        self._check_tensor(name, env_mask, self.torch.bool, (self.num_envs,))
        return env_mask.contiguous()

    @staticmethod
    def _task_key(slot, d):
        return (slot, np.asarray(d["rand_vec"], dtype=np.float64).tobytes(), bool(d["partially_observable"]))

    def _ensure_snapshots(self, tasks):
        """Episode-start snapshots for tasks the engine has not seen yet (construction, checkpoints with other goals)."""
        mi, rvs, po, keys = [], [], [], []
        for tk in tasks:
            d = tk.unpack()
            key = self._task_key(self._slot_of_name[tk.env_name], d)
            if key in self._snap_of or key in keys:
                continue
            v = np.asarray(d["rand_vec"], dtype=np.float64)
            rv = np.zeros(6)
            rv[: len(v)] = v
            keys.append(key); mi.append(key[0]); rvs.append(rv); po.append(key[2])
            self._task_of_snap[key] = tk
        if keys:
            ids = self.engine.build_snapshots(mi, np.array(rvs), po)
            for k, i in zip(keys, ids):
                self._snap_of[k] = int(i)
                self._task_of_snap[int(i)] = self._task_of_snap.pop(k)

    def _snap(self, task: Task) -> int:
        i = task.__dict__.get("_snap_id")
        if i is None or task.__dict__.get("_snap_owner") is not self:
            i = self._snap_of[self._task_key(self._slot_of_name[task.env_name], task.unpack())]
            task.__dict__["_snap_id"], task.__dict__["_snap_owner"] = i, self
        return i

    def _push_next(self):
        self.h_next.copy_(self.torch.from_numpy(self._next_ids))
        self.d_next.copy_(self.h_next, non_blocking=True)

    def _draw_pending(self, e):
        s = self.sub[e]
        s.draw_pending()
        self._next_ids[e] = self._snap(s.pending)

    def _redraw_all_pending(self):
        for e, s in enumerate(self.sub):
            s.rewind_pending()
            self._draw_pending(e)
        self._push_next()

    def _take_reset_draws(self, idx):
        """The task-select draw of `reset` for sub-envs `idx`: the snapshot ids of their new episodes go to `d_cur` (other
        rows 0) and the draws for the episodes after them to `d_next`.  Each sub-env has its own RNG, so the order across
        envs does not matter."""
        cur = np.zeros(self.num_envs, dtype=np.int32)
        for e in idx:
            s = self.sub[e]
            s.take_for_reset()
            cur[e] = self._snap(s.current_task)
            self._draw_pending(e)
        self.d_cur.copy_(self.torch.from_numpy(cur))
        self._push_next()

    # ------------------------------------------------------------------ VectorEnv API
    def reset(self, *, seed=None, options=None):
        """Every sub-env: (task-select wrapper) pick a task, then SawyerXYZEnv.reset (its `seed` argument is ignored,
        sawyer_xyz_env.py:670).  ``options={"reset_mask": m}`` (numpy bool [num_envs], any mode) resets only the envs
        with ``m`` set; the other rows of the returned observation are the ones the previous call returned for them."""
        if options is not None and "reset_mask" in options:
            return self._reset_masked(options["reset_mask"])
        self._take_reset_draws(range(self.num_envs))
        self.engine.reset(self.d_cur, self.d_obs)
        self._d_raw = self.d_obs
        self._ep_len[:] = 0
        self._needs_reset = False
        self.h_obs.copy_(self.d_obs)
        obs = self.h_obs.numpy().astype(self.obs_dtype)
        self._obs_template = obs.copy()        # constant columns (one-hot task id) of every later observation; see step()
        self._obs_template[:, :39] = 0
        self._autoreset_envs.set(host=np.zeros(self.num_envs, dtype=bool))
        if self.post.active:
            obs = self.post.on_reset(obs)
        self._returned_obs.set(host=obs, device=None if self.post.active else self.d_obs)   # (d_obs: the same values)
        return obs, {}

    def _reset_masked(self, mask):
        """gymnasium's `reset(options={"reset_mask": mask})`: the masked envs take their task-select draw and restart
        (k_reset_masked); infos are merged for them only, and the reset info is empty."""
        N = self.num_envs
        assert isinstance(mask, np.ndarray), f"`options['reset_mask': mask]` must be a numpy array, got {type(mask)}"
        assert mask.shape == (N,), f"`options['reset_mask': mask]` must have shape `({N},)`, got {mask.shape}"
        assert mask.dtype == np.bool_, f"`options['reset_mask': mask]` must have `dtype=np.bool_`, got {mask.dtype}"
        assert np.any(mask), f"`options['reset_mask': mask]` must contain a boolean array, got reset_mask={mask}"
        if self._needs_reset:
            raise RuntimeError("reset() without a mask must come first")
        if self._device_sampler:
            raise RuntimeError("the device-side task sampler is active (step_torch was used): use reset_torch(reset_mask) or "
                               "disable_device_sampler() + reset()")
        if not self._returned_obs.on_host():
            raise RuntimeError("the last observations are on the device (step_torch): use reset_torch(reset_mask=...)")
        idx = np.nonzero(mask)[0]
        self._take_reset_draws(idx)
        d_mask = self.torch.from_numpy(mask).to(self.device)
        self.engine.reset_masked(d_mask, self.d_obs, self.d_cur)
        self._merge_raw_rows(d_mask)
        self.h_obs.copy_(self.d_obs)
        rows = self.h_obs.numpy()[idx].astype(self.obs_dtype)
        self._ep_len[idx] = 0
        self._autoreset_envs.host(write=True)[idx] = False
        obs = self._returned_obs.host().copy()
        if self.post.active:
            full = np.zeros((N, rows.shape[1]), dtype=self.obs_dtype)
            full[idx] = rows
            rows = self.post.on_reset(full, mask)[idx]
        obs[idx] = rows
        self._returned_obs.set(host=obs)
        return obs, {}

    def _merge_raw_rows(self, d_mask):
        """After a masked reset into `d_obs`: when the other envs' base observations are in `d_obs39` (the last call was
        the numpy `step`), the reset rows join them there."""
        if self._d_raw is self.d_obs39:
            self.d_obs39.copy_(self.torch.where(d_mask[:, None], self.d_obs[:, :39], self.d_obs39))

    def _advance_streams(self, idx):
        """The autoreset's task-select draw of sub-envs `idx` (their episode ends with this step): the speculative draw
        becomes the running task and the draw for the episode after it is made."""
        for e in idx:
            s = self.sub[e]
            s.current_task, s._pre = s.pending, None
            self._draw_pending(e)
        self._push_next()

    def step(self, actions):
        if self._needs_reset:
            raise RuntimeError("reset() must be called before step()")
        if self._device_sampler:
            raise RuntimeError("the device-side task sampler is active (step_torch was used): the numpy step API and its host "
                               "task streams are no longer in sync; call disable_device_sampler() + reset() first")
        if self.autoreset_mode != "SameStep":
            return self._step_deferred(actions)
        N = self.num_envs
        a, pred = self._launch(actions)
        # while the kernel runs: the task streams of the envs it truncates are advanced and the snapshot ids of the episodes
        # after the coming ones are queued behind it (stream order: k_step reads d_next before this copy overwrites it)
        if len(pred):
            self._advance_streams(pred)
        obs, sm, reward, terminated, truncated = self._collect()
        done = terminated | truncated
        idx = np.nonzero(done)[0]
        any_done = len(idx) > 0
        # SAME_STEP (gymnasium SyncVectorEnv): a finished env's step info moves to `final_info` and its slot in the
        # top-level arrays is the (empty) reset info
        infos = self._step_infos(sm, idx)
        fo = ep_r = None
        if any_done:
            # terminal observations / infos of the finished envs only (a few rows per step in steady state)
            rows_o = self._obs_template[idx]
            rows_o[:, :39] = self._terminal_rows(idx, pred, self.h_final_obs39, self.d_final_obs39)
            rows_i = self._terminal_rows(idx, pred, self.h_final_info, self.d_final_info)
        if self.post.active:
            if any_done:
                fo = np.zeros((N, self.obs_dim), dtype=self.obs_dtype)
                fo[idx] = rows_o
            obs, reward, fo, ep_r = self.post.on_step(obs, a, reward, terminated, truncated, final_obs=fo)
            if any_done:
                rows_o = fo[idx]
        if any_done:
            fi = np.zeros((8, N))
            fi[:, idx] = rows_i.T
            if ep_r is not None:
                fi[7] = ep_r             # RecordEpisodeStatistics sits outside the reward normalisation
            final_obs = np.full(N, None, dtype=object)
            for j, e in enumerate(idx):
                final_obs[e] = rows_o[j]
            final_info = {}
            for i, k in enumerate(INFO_KEYS):
                final_info[k] = fi[i]                              # rows of unfinished envs are 0
                final_info["_" + k] = done.copy()
            final_info["episode"], final_info["_episode"] = self._episode_stats(done, fi[7])
            infos["final_obs"], infos["_final_obs"] = final_obs, done.copy()
            infos["final_info"], infos["_final_info"] = final_info, done.copy()
            self._ep_len[idx] = 0
            if len(pred) < len(idx):                 # terminations nobody could predict (terminate_on_success)
                self._advance_streams(np.setdiff1d(idx, pred))
        self._returned_obs.set(host=obs)
        return obs, reward, terminated, truncated, infos

    def _step_deferred(self, actions):
        """`step` under NEXT_STEP / DISABLED autoreset (gymnasium SyncVectorEnv): the terminal step returns the terminal
        observation and the step infos of every env, with RecordEpisodeStatistics' `episode` at the top level.  NEXT_STEP:
        the next call restarts the envs that ended (their action is ignored) and returns their reset observation with
        reward 0, no flags and no infos; their task-select draw becomes the running task then.  DISABLED: stepping an env
        that ended and was not reset (`reset(options={"reset_mask": ...})`) fails before anything is launched."""
        N = self.num_envs
        ended = self._autoreset_envs.host()
        if self.autoreset_mode == "Disabled":
            assert not ended.any(), f"self._autoreset_envs={ended!r}"      # SyncVectorEnv's DISABLED assertion
        restart = np.nonzero(ended)[0]      # (none under DISABLED)
        a, pred = self._launch(actions, ended)
        if len(restart):                 # queued behind the kernel, which has read these envs' snapshot ids
            self._advance_streams(restart)
        obs, sm, reward, terminated, truncated = self._collect()
        self._ep_len[restart] = 0
        done = terminated | truncated
        idx = np.nonzero(done)[0]
        infos = self._step_infos(sm, restart)
        ep_r = None
        if self.post.active:
            fresh = np.zeros(N, dtype=bool)
            fresh[restart] = True
            obs, reward, _, ep_r = self.post.on_step(obs, a, reward, terminated, truncated, restart=fresh)
        if len(idx):
            if ep_r is None:
                ep_r = np.zeros(N)
                ep_r[idx] = self._terminal_rows(idx, pred, self.h_final_info[:, 7], self.d_final_info[:, 7])
            infos["episode"], infos["_episode"] = self._episode_stats(done, ep_r)
        self._autoreset_envs.set(host=done)
        self._returned_obs.set(host=obs)
        return obs, reward, terminated, truncated, infos

    def _launch(self, actions, ended=None):
        """Uploads `actions`, launches k_step and queues the copies of its results behind it: the packed [N, 9] record,
        the 39 observation columns it writes, and the terminal rows of the envs whose episode it truncates.  Those are known
        in advance (the host mirrors the episode lengths), so on most steps one synchronise brings back everything.
        `ended` (NEXT_STEP / DISABLED): the envs that ended in the previous call, which restart or stand still.
        -> (the actions as a float32 [N, 4] array, the indices of those envs)"""
        t = self.torch
        a = np.ascontiguousarray(actions, dtype=np.float32).reshape(self.num_envs, 4)
        self.h_actions.copy_(t.from_numpy(a))
        self.d_actions.copy_(self.h_actions, non_blocking=True)
        self.engine.step(self.d_actions, self.d_obs39, self.d_reward, self.d_term, self.d_trunc, self.d_small,
                         self.d_final_obs39, self.d_final_info, self.d_next)
        self._d_raw = self.d_obs39
        self.h_small.copy_(self.d_small, non_blocking=True)
        self.h_obs39.copy_(self.d_obs39, non_blocking=True)
        due = self._ep_len + 1 >= min(self.max_episode_steps, MAX_PATH_LENGTH)
        pred = np.nonzero(due if ended is None else due & ~ended)[0]
        npred = len(pred)
        if npred:
            self.h_idx[:npred] = t.from_numpy(pred)
            d_pred = self.d_idx[:npred]
            d_pred.copy_(self.h_idx[:npred], non_blocking=True)
            # (only SAME_STEP writes terminal observations; copying their rows in every mode keeps a single path)
            self.h_final_obs39[:npred].copy_(self.d_final_obs39.index_select(0, d_pred), non_blocking=True)
            self.h_final_info[:npred].copy_(self.d_final_info.index_select(0, d_pred), non_blocking=True)
        return a, pred

    def _collect(self):
        """Waits for the step `_launch` queued and counts it in `_ep_len`.
        -> (a fresh observation array, the packed record as [9, N] float64 rows, reward, terminated, truncated)"""
        # fresh arrays every step, like the reference (:637).  The array is allocated before the synchronise, as a copy of
        # a template that already holds the constant columns (the one-hot task id): only the 39 columns the kernel writes
        # remain to be converted once the results are there
        obs = self._obs_template.copy()
        if self.device.type == "cuda":
            self.torch.cuda.current_stream(self.device).synchronize()
        # ---- results (single-threaded numpy on purpose: torch's parallel host copies are faster when idle but collapse
        # under a cgroup CPU quota smaller than the machine's core count)
        np.copyto(obs[:, :39], self.h_obs39.numpy())
        sm = np.ascontiguousarray(self.h_small.numpy().T, dtype=np.float64)      # [9, N]: rows are contiguous per-key arrays
        flags = sm[8].astype(np.int8)
        self._ep_len += 1
        return obs, sm, sm[7], (flags & 1).astype(bool), (flags & 2).astype(bool)

    def _step_infos(self, sm, blank):
        """The top-level step infos from the packed record's rows `sm`.  The envs `blank` report the (empty) reset info
        instead: value 0, mask False; the keys vanish when every env does."""
        infos = {}
        if len(blank) < self.num_envs:
            live = np.ones(self.num_envs, dtype=bool)
            live[blank] = False
            for i, k in enumerate(INFO_KEYS):
                v = sm[i]
                v[blank] = 0.0
                infos[k] = v
                infos["_" + k] = live.copy()
        return infos

    def _terminal_rows(self, idx, pred, h_rows, d_rows):
        """Rows `idx` of the device array `d_rows`: those `_launch` copied to `h_rows` when `idx` is exactly the predicted
        truncations `pred` (always, unless success terminates an episode), otherwise fetched now."""
        if np.array_equal(idx, pred):
            return h_rows[:len(pred)].numpy()
        return d_rows.index_select(0, self.torch.from_numpy(idx).to(self.device)).cpu().numpy()

    def _episode_stats(self, done, returns):
        """RecordEpisodeStatistics' `episode` entry and `_episode` mask for the envs that finished (`done`)."""
        return ({"r": returns, "l": np.where(done, self._ep_len, 0), "t": np.zeros(self.num_envs),
                 "_r": done.copy(), "_l": done.copy(), "_t": done.copy()}, done.copy())

    def step_async(self, actions):
        self._pending_actions = actions

    def step_wait(self):
        return self.step(self._pending_actions)

    # GPU-resident variants (no host synchronisation; task re-sampling on autoreset happens on the device).  The optional
    # recurrent-obs / normalisation wrappers are applied on the device as well, by the same `post.StepPost` as `step`.
    def enable_device_sampler(self):
        """Autoreset draws the next goal on the device: uniform over the env's own task list, a counter-based hash of
        (seed, env, episode) -- the distribution of RandomTaskSelectWrapper, not its PCG64 stream.  The host task mirrors
        stop being advanced; `get_attr("_last_rand_vec")` etc. then read the snapshot id back from the device."""
        first, count = [], []
        for e, s in enumerate(self.sub):
            ids = sorted(self._snap(tk) for tk in s.tasks)
            assert ids == list(range(ids[0], ids[0] + len(ids))), "device sampler needs contiguous snapshot ranges"
            first.append(ids[0]); count.append(len(ids))
        self.engine.set_goal_sets(first, count)
        self._device_sampler = True

    def disable_device_sampler(self):
        self._device_sampler = False
        self._needs_reset = True

    def reset_torch(self, reset_mask=None):
        """Without a mask: `reset()`, result on the device.  `reset_mask` (bool CUDA tensor [num_envs]): only those envs
        restart, as `reset(options={"reset_mask": ...})` does, without host synchronisation: their snapshot comes from the
        device sampler (or the pre-drawn task when no env re-samples), and the other rows are what the previous call
        returned.  The returned tensor is overwritten by the next call."""
        if reset_mask is None:
            self.reset()      # with the optional wrappers: their reset() output, so their statistics see it only once
            return self._returned_obs.device()
        if self._needs_reset:
            raise RuntimeError("reset_torch() without a mask must come first")
        mask = self._torch_mask(reset_mask, "reset_mask")
        if not self._device_sampler and any(s.sample_tasks_on_reset for s in self.sub):
            self.enable_device_sampler()
        last = self._returned_obs.device()
        self.engine.reset_masked(mask, self.d_obs, None if self._device_sampler else self.d_next)
        return self._restarted(mask, last)

    def _restarted(self, mask, last):
        """The bookkeeping of a masked restart into `d_obs` (bool device tensor `mask`) from the observations `last` the
        previous call returned, on the device (taken before the restart: without the optional wrappers they are `d_obs`):
        base rows, ended marks, the optional wrappers' reset; returns the observations as `reset_torch(mask)` does."""
        self._merge_raw_rows(mask)
        self._autoreset_envs.device(write=True).logical_and_(~mask)
        out = self.torch.where(mask[:, None], self.post.on_reset(self.d_obs, mask), last) if self.post.active else last
        self._returned_obs.set(device=out)
        return out

    def step_torch(self, actions):
        """`actions`: float32 CUDA tensor [num_envs, 4] on this env's device.  Returns device tensors (obs [N, obs_dim],
        reward [N], terminated u8 [N], truncated u8 [N], info [N, 7]) that are overwritten by the next call."""
        t = self.torch
        if self._needs_reset:
            raise RuntimeError("reset() must be called before step_torch()")
        self._check_tensor("actions", actions, t.float32, (self.num_envs, 4), contiguous=True)
        if not self._device_sampler and any(s.sample_tasks_on_reset for s in self.sub):
            self.enable_device_sampler()      # without it every autoreset would restart the same pre-drawn goal
        nxt = None if self._device_sampler else self.d_next
        ended = restart = None
        if self.autoreset_mode != "SameStep":      # NEXT_STEP restarts the envs that ended in the previous call
            ended = self._autoreset_envs.device(write=True)
            restart = ended.clone() if self.autoreset_mode == "NextStep" else None
        self.engine.step(actions, self.d_obs, self.d_reward, self.d_term, self.d_trunc, self.d_small, self.d_final_obs,
                         self.d_final_info, nxt)
        self._d_raw = self.d_obs
        if ended is not None:
            t.logical_or(self.d_term, self.d_trunc, out=ended)
        obs, rew = self.d_obs, self.d_reward
        if self.post.active:       # the optional wrappers on the device; the terminal observation and episode returns stay available
            obs, rew, self.d_final_obs_post, self.d_episode_return_post = self.post.on_step(
                self.d_obs, actions, self.d_reward, self.d_term, self.d_trunc,
                self.d_final_obs if self.autoreset_mode == "SameStep" else None, restart=restart)
        self._returned_obs.set(device=obs)
        return obs, rew, self.d_term, self.d_trunc, self.d_info

    # ------------------------------------------------------------------ physics state (MujocoEnv.set_state, get_env_state, _get_obs)
    # The optional wrappers are not involved: the reference's `call` reaches these methods on the base env.
    def _check_started(self, what):
        if self._needs_reset:
            raise RuntimeError(f"reset() must be called before {what} (the device state is created by reset)")

    def set_state(self, qpos, qvel, env_mask=None):
        """MujocoEnv.set_state for the envs with `env_mask` set (numpy bool [num_envs]; None = all): `qpos` [num_envs, 18]
        and `qvel` [num_envs, 17] (numpy, the layout of `get_state_torch`; columns past an env's nq / nv are ignored).  qvel
        is stored as float32.  Only the physics state changes: the observation is what `observe` computes from it, and an
        ended env (NEXT_STEP / DISABLED) restarts from its next task as usual, overwriting the state."""
        self._check_started("set_state")
        N = self.num_envs
        qpos, qvel = np.asarray(qpos, dtype=np.float64), np.asarray(qvel, dtype=np.float64)
        if qpos.shape != (N, MAXNQ) or qvel.shape != (N, MAXDOF):
            raise ValueError(f"set_state needs qpos of shape ({N}, {MAXNQ}) and qvel of shape ({N}, {MAXDOF}), got {qpos.shape} and {qvel.shape}")
        rows = self._host_mask(env_mask)
        nq, nv = self._getters.dims()
        used_q = (np.arange(MAXNQ) < nq[:, None]) & rows[:, None]
        used_v = (np.arange(MAXDOF) < nv[:, None]) & rows[:, None]
        if not (np.isfinite(qpos[used_q]).all() and np.isfinite(qvel[used_v]).all()):
            raise ValueError("set_state: qpos / qvel of the selected envs must be finite")
        t = self.torch
        self.set_state_torch(t.from_numpy(np.ascontiguousarray(qpos)).to(self.device),
                             t.from_numpy(np.ascontiguousarray(qvel)).to(self.device), self._device_mask(env_mask))

    def set_state_torch(self, qpos, qvel, env_mask=None):
        """`set_state` from device tensors, without host synchronisation: `qpos` float64 [num_envs, 18], `qvel` float64
        [num_envs, 17], contiguous, on this env's device; `env_mask` a bool tensor [num_envs] or None (all).  Values are not
        inspected (a non-finite state shows up as a non-finite observation fault)."""
        self._check_started("set_state_torch")
        self._check_tensor("qpos", qpos, self.torch.float64, (self.num_envs, MAXNQ), contiguous=True)
        self._check_tensor("qvel", qvel, self.torch.float64, (self.num_envs, MAXDOF), contiguous=True)
        self.engine.set_physics(self._torch_mask(env_mask), qpos, qvel)

    def get_state_torch(self):
        """Every env's (qpos float64 [num_envs, 18], qvel float64 [num_envs, 17]) as new device tensors, without host
        synchronisation; columns past an env's nq / nv are zero.  `set_state_torch` takes them back."""
        self._check_started("get_state_torch")
        t = self.torch
        qpos = t.empty(self.num_envs, MAXNQ, dtype=t.float64, device=self.device)
        qvel = t.empty(self.num_envs, MAXDOF, dtype=t.float64, device=self.device)
        self.engine.get_physics(qpos, qvel)
        return qpos, qvel

    def observe_torch(self, env_mask=None):
        """SawyerXYZEnv._get_obs() of the current state for the envs with `env_mask` set (bool tensor [num_envs]; None =
        all), with their one-hot columns when `use_one_hot`: the frame-stacked observation, unclipped, not passed through the
        optional wrappers.  Like the reference it makes the current frame the env's previous one (the next step's
        obs[18:36]).  Returns a float32 device tensor [num_envs, obs_dim] that the next call overwrites; rows of the
        other envs are what the previous call left there (zero before the first)."""
        self._check_started("observe_torch")
        self.engine.observe(self._torch_mask(env_mask), self.d_env_obs)
        return self.d_env_obs

    def observe(self, env_mask=None):
        """`observe_torch` with a numpy bool mask (None = all); a float64 numpy array [num_envs, obs_dim]."""
        self._check_started("observe")
        return self.observe_torch(self._device_mask(env_mask)).cpu().numpy().astype(np.float64)

    # ------------------------------------------------------------------ saved states (save, restore and fork on the device)
    # A loaded env continues bit for bit as its source would have, up to the end of the current episode, in every autoreset
    # mode.  The task-selection streams (host RNGs, the pending draw, the device sampler's key) are not part of a state:
    # each env keeps its own, and `get_checkpoint` saves them.  Across a restart the replay is exact when the env draws
    # the same snapshot as its source: always with the device sampler and `src` = identity (it keys on seed, env and
    # the restored episode counter), and whenever `sample_tasks_on_reset` is False.  Fault bits, counters, profiles and
    # the launch order are not part of a state.
    def save_states(self, env_mask=None):
        """An `EnvStates` with the complete state of every env with `env_mask` set (numpy or device bool [num_envs]; None =
        all), without host synchronisation (with a numpy mask: one upload)."""
        self._check_started("save_states")
        t, N = self.torch, self.num_envs
        if env_mask is not None:
            env_mask = self._torch_mask(env_mask) if isinstance(env_mask, t.Tensor) else self._device_mask(env_mask)
        records = t.zeros(N, 512, dtype=t.uint8, device=self.device)
        model = t.full((N,), -1, dtype=t.int32, device=self.device)
        hints = t.zeros(N, NCONV, 4, dtype=t.float32, device=self.device)
        self.engine.save_states(records, model, hints, env_mask)
        obs = self._returned_obs.host().copy() if self._returned_obs.on_host() else self._returned_obs.device().clone()
        return EnvStates(self, records, model, hints, self._d_raw[:, :39].clone(), obs,
                         self.post.save_rows() if self.post.active else None, self._ep_len.copy(),
                         [s.current_task for s in self.sub], None if self._goal_bufs is None else self._goal_bufs[2].clone())

    def _check_states(self, states, what):
        self._check_started(what)
        if not isinstance(states, EnvStates) or states.owner is not self:
            raise ValueError(f"{what}: the states were saved by another env (snapshot ids are engine-local)")

    def _restore_mirrors(self, rows, ep_len, tasks):
        """The host mirrors of envs `rows` as a saved state has them: episode lengths and running tasks."""
        self._ep_len[rows] = ep_len
        for e, tk in zip(rows, tasks):
            self.sub[e].current_task = tk

    def load_states(self, states, env_mask=None, src=None):
        """Env e with `env_mask[e]` set (numpy bool [num_envs]; None = all) takes row `src[e]` (numpy integers [num_envs];
        None = row e) of `states`, which this env saved.  A source row out of range, unsaved or of another model raises
        ValueError before anything changes.  Returns the observations as `reset(options={"reset_mask": ...})` does: the
        loaded envs' saved last observation, the other envs' last one.  Sub-envs that do not re-sample their task on
        reset continue with the loaded task after the episode; the others keep their own task streams."""
        self._check_states(states, "load_states")
        N = self.num_envs
        mask = self._host_mask(env_mask)
        src = np.arange(N) if src is None else np.asarray(src)
        if src.shape != (N,) or src.dtype.kind not in "iu":
            raise ValueError(f"src must be a numpy integer array of shape ({N},)")
        src = np.where(mask, src, np.arange(N))         # unmasked rows: never read, kept in range for the row gathers below
        rows = np.nonzero(mask)[0]
        s = src[rows]
        bad = rows[(s < 0) | (s >= N)]
        if not len(bad):
            bad = rows[states.model.cpu().numpy()[s] != self._env_model[rows]]
        if len(bad):
            raise ValueError(f"load_states: env(s) {bad.tolist()[:8]} have no saved state of their model at the given src")
        t = self.torch
        self.load_states_torch(states, t.from_numpy(mask).to(self.device), t.from_numpy(src.astype(np.int32)).to(self.device))
        self._restore_mirrors(rows, states.ep_len[s], [states.tasks[i] for i in s])
        for e in rows:
            if not self.sub[e].sample_tasks_on_reset:
                self._draw_pending(e)
        self._push_next()
        self._autoreset_envs.host()        # fetched here, not by the next numpy `step`
        return self._returned_obs.host()

    def load_states_torch(self, states, env_mask=None, src=None):
        """`load_states` from device tensors, without host synchronisation: `env_mask` a bool tensor [num_envs] or None (all),
        `src` an integer tensor [num_envs] or None (row e).  An env whose source row is out of range, unsaved or of another
        model is left unchanged and gets fault bit 32 (`engine.raise_on_faults()` raises ValueError).  The host mirrors
        (episode lengths, running tasks) are left as they are, as `step_torch` leaves them.  Returns the observations as
        `reset_torch(mask)` does: the loaded envs' saved last observation, the other envs' last one."""
        self._check_states(states, "load_states_torch")
        t, N = self.torch, self.num_envs
        mask = self._torch_mask(env_mask)
        if src is None:
            src = t.arange(N, device=self.device)
        else:
            self._check_tensor("src", src, "integer", (N,))
        src = src.long()
        sc = src.clamp(0, N - 1)
        ok = mask & (src >= 0) & (src < N) & (states.model[sc] == self.d_env_model)    # the check of k_load_states
        self.engine.load_states(states.records, states.model, states.hints, None if env_mask is None else mask,
                                src.to(t.int32))
        if self.autoreset_mode != "SameStep":
            ended = self._autoreset_envs.device(write=True)
            ended.copy_(t.where(ok, states.ended()[sc], ended))
        self._d_raw[:, :39] = t.where(ok[:, None], states.raw[sc], self._d_raw[:, :39])
        self._load_goals(states, ok, sc)
        saved = states.obs
        if isinstance(saved, np.ndarray):          # saved right after a numpy call
            saved = t.from_numpy(saved.astype(np.float32)).to(self.device)
        out = t.where(ok[:, None], saved[sc], self._returned_obs.device())
        if self.post.active:
            self.post.load_rows(states.post, ok, sc)
        else:
            out = self.d_obs.copy_(out)
        self._returned_obs.set(device=out)
        return out

    def _load_goals(self, states, mask, src):
        """The running goals of a load: env e takes row `src[e]` of the saved goal table where `mask[e]` (device tensors)."""
        if states.goal is not None:
            goal = self._goal_buffers()[2]
            goal.copy_(self.torch.where(mask[:, None], states.goal[src], goal))

    # ------------------------------------------------------------------ episodes at new goals (unfrozen rand_vec)
    # `reset_goals_torch(g, m)` is `engine.reset_masked(m, obs, ids)` with `ids` the snapshots of the goals `g`, except that
    # no snapshot is built or stored and the records' snapshot id is -1.  No task-selection draw is consumed: the pending
    # draw stays pending, and the device sampler draws for the next episode as for any other.  The goal an env runs on is
    # part of its state until its next reset: `get_attr("_last_rand_vec")`, `save_states` / `load_states` and the
    # checkpoints carry it.
    def _goal_buffers(self):
        """(goal rows uint8 [N, 768], observability uint8 [N], running goals float64 [N, 6]) on the device."""
        if self._goal_bufs is None:
            t, N = self.torch, self.num_envs
            self._goal_bufs = (t.zeros(N, SNAPSHOT_DTYPE.itemsize, dtype=t.uint8, device=self.device),
                               t.from_numpy(self._partial.astype(np.uint8)).to(self.device),
                               t.zeros(N, 6, dtype=t.float64, device=self.device))
        return self._goal_bufs

    def reset_goals_torch(self, rand_vec, env_mask=None, rand_vec_pass1=None):
        """Restarts the envs with `env_mask` set (bool CUDA tensor [num_envs]; None = all) at the goals `rand_vec` (float64
        CUDA tensor [num_envs, 6]: each env's `_last_rand_vec`, in the leading columns when its task's is shorter), as a
        reset with an unfrozen rand_vec does: the reference's reset() with `rand_vec_pass1` (same layout; None = `rand_vec`)
        in the first reset_model pass.  Works in every autoreset mode, without host synchronisation; returns the
        observations as `reset_torch(mask)` does.  An env whose goal is not finite is left as it is and gets fault bit 64
        (`engine.raise_on_faults()` raises ValueError)."""
        t, N = self.torch, self.num_envs
        if self._needs_reset:
            raise RuntimeError("reset() must be called before reset_goals_torch()")
        self._check_tensor("rand_vec", rand_vec, t.float64, (N, 6))
        if rand_vec_pass1 is not None:
            self._check_tensor("rand_vec_pass1", rand_vec_pass1, t.float64, (N, 6))
        mask = self._torch_mask(env_mask)
        rows, partial, goal = self._goal_buffers()
        rv = rand_vec.contiguous()
        self.engine.build_goal_rows(mask, rv, None if rand_vec_pass1 is None else rand_vec_pass1.contiguous(), partial, rows)
        last = self._returned_obs.device()
        self.engine.reset_rows(mask, rows, self.d_obs)
        f = rows.view(t.float32)                   # the envs k_reset_rows restarted: finite goal and observation
        ok = mask & t.isfinite(f[:, _ROW_OBS:_ROW_OBS + 39]).all(1) & t.isfinite(f[:, _ROW_TARGET:_ROW_TARGET + 3]).all(1)
        goal.copy_(t.where(ok[:, None], rv, goal))
        return self._restarted(ok, last)

    def reset_goals(self, rand_vec, env_mask=None, rand_vec_pass1=None):
        """`reset_goals_torch` from numpy: `rand_vec` (and `rand_vec_pass1`) float64 [num_envs, 6], `env_mask` numpy bool
        [num_envs] or None (all).  Shapes, dtypes, the mask and the finiteness of the masked rows are checked before
        anything changes (ValueError).  Returns the observations as `reset(options={"reset_mask": ...})` does: the new
        episodes' first observations in the masked rows, the last ones returned in the others."""
        N = self.num_envs
        mask = self._host_mask(env_mask)
        vecs = []
        for name, x in (("rand_vec", rand_vec), ("rand_vec_pass1", rand_vec_pass1)):
            if x is None and name == "rand_vec_pass1":
                vecs.append(None)
                continue
            a = np.asarray(x)
            if a.shape != (N, 6) or a.dtype != np.float64:
                raise ValueError(f"reset_goals needs {name} as a float64 array of shape ({N}, 6), got {a.dtype} {a.shape}")
            if not np.isfinite(a[mask]).all():
                raise ValueError(f"reset_goals: {name} has non-finite entries in the rows of masked envs")
            vecs.append(a)
        if self._needs_reset:
            raise RuntimeError("reset() must be called before reset_goals()")
        t = self.torch
        obs = self._returned_obs.host().copy()
        d = [None if a is None else t.from_numpy(np.ascontiguousarray(a)).to(self.device) for a in vecs]
        out = self.reset_goals_torch(d[0], t.from_numpy(mask).to(self.device), d[1])
        idx = np.nonzero(mask)[0]
        self._ep_len[idx] = 0
        self._autoreset_envs.host()        # fetched here, not by the next numpy `step`
        obs[idx] = out.cpu().numpy()[idx]
        self._returned_obs.set(host=obs)
        return obs

    def sample_goals(self, rng, env_mask=None):
        """Goals for `reset_goals`: for every env with `env_mask` set (numpy bool [num_envs]; None = all), in env order,
        the two draws of a reset with an unfrozen rand_vec (`benchmarks.draw_rand_vec`: each env's task's
        _random_reset_space and rejection loop) from `rng`, a numpy Generator or RandomState.  Returns numpy float64
        (rand_vec, rand_vec_pass1) [num_envs, 6]; other rows are zero."""
        N = self.num_envs
        mask = self._host_mask(env_mask)
        rv, rv1 = np.zeros((N, 6)), np.zeros((N, 6))
        for e in np.nonzero(mask)[0]:
            spec = TASKS[self.sub[e].task_name]
            first = draw_rand_vec(spec, rng)
            second = draw_rand_vec(spec, rng)
            rv1[e, :first.size], rv[e, :second.size] = first, second
        return rv, rv1

    def _goal_task(self, e, v):
        """The Task of env e's running episode on goal `v` (a reset_goals row)."""
        name = self.sub[e].task_name
        return make_task(name, np.array(v[:TASKS[name].rand_low.size], dtype=np.float64), bool(self._partial[e]))

    # ------------------------------------------------------------------ state accessors (SawyerXYZEnv / MujocoEnv getters)
    def query_torch(self, env_mask=None, bodies=(), sites=(), geoms=(), touching=False):
        """Read-only accessors of every env's current state (envs with `env_mask` set; bool tensor [num_envs], None =
        all), as a dict of new device tensors, without host synchronisation and without changing any state:

        * ``frame``: float32 [num_envs, 18], columns 0..17 of the next `observe_torch` (hand, gripper distance, the 14
          object slots), unclipped; the frame stack is not advanced.
        * ``body_xpos`` / ``body_xquat`` (float64 [num_envs, len(bodies), 3] / [.., 4], w x y z), ``site_xpos`` /
          ``site_xmat`` ([.., 3] / [.., 3, 3]) and ``geom_xpos`` / ``geom_xmat``: MuJoCo's data.body / site / geom(name)
          poses; a name an env's model lacks gives NaN.
        * ``touching`` (when `touching`): bool [num_envs], the reference's ``touching_main_object`` for the geom its
          ``_get_id_main_object`` names, False where that returns None.  Runs the full forward pass (contact forces).

        Rows of the other envs are zero (their ``*_xmat`` rows: the identity, the matrix of a zero quaternion)."""
        self._check_started("query_torch")
        mask = self._torch_mask(env_mask)
        for kind, names in (("body", bodies), ("site", sites), ("geom", geoms)):
            if isinstance(names, str) or not all(isinstance(n, str) for n in names):
                raise ValueError(f"query_torch: {kind}s must be a sequence of {kind} names")
        return self._getters.query(mask, bodies, sites, geoms, touching)

    # ------------------------------------------------------------------ scripted experts (metaworld.policies)
    def expert_actions_torch(self, obs=None):
        """Every env's scripted expert action (metaworld_b200.policies: its task's policy in ENV_POLICY_MAP), as a new
        float32 device tensor [num_envs, 4], unclipped, without host synchronisation.  `obs=None` reads each env's base
        observation as the last `reset` / `step` / `reset_torch` / `step_torch` left it, before the optional wrappers
        (normalisation, recurrent info), which the policies never see; on a NEXT_STEP / DISABLED terminal step that is
        the terminal observation.  Otherwise `obs` is a float32 device tensor [num_envs, >= 39] whose first 39 columns
        are base observations, e.g. `observe_torch()` after `set_state_torch`; later columns (one-hot ids) are ignored."""
        t = self.torch
        if obs is None:
            self._check_started("expert_actions_torch")
            obs = self._d_raw
        else:
            self._check_tensor("obs", obs, t.float32, (self.num_envs,), min_cols=39)
        if self._d_expert_ids is None:
            self._d_expert_ids = t.tensor([TASK_IDS.get(s.task_name, -1) for s in self.sub], dtype=t.int32, device=self.device)
        out = t.empty(self.num_envs, 4, dtype=t.float32, device=self.device)
        expert_actions(self._d_expert_ids, obs, out)
        return out

    def expert_actions(self, obs=None):
        """`expert_actions_torch` as a float32 numpy array [num_envs, 4]; `obs` None or a numpy array [num_envs, >= 39]."""
        if obs is not None:
            o = np.asarray(obs)
            if o.ndim != 2 or o.shape[0] != self.num_envs or o.shape[1] < 39:
                raise ValueError(f"expert_actions needs obs of shape ({self.num_envs}, >= 39), got {o.shape}")
            obs = self.torch.from_numpy(np.ascontiguousarray(o[:, :39], dtype=np.float32)).to(self.device)
        return self.expert_actions_torch(obs).cpu().numpy()

    # ------------------------------------------------------------------ open-loop rollouts (planning)
    # A rollout answers "from where each env is now, what would each of these K action sequences earn over H steps?"
    # without moving the envs.  Each step is `step_torch`'s step of the base env, bit for bit, with TimeLimit and
    # terminate_on_success; a row's episode end is its last live step (no autoreset, no task draw).  The optional
    # wrappers and one-hot columns are not applied, as in `observe_torch` and `expert_actions_torch`.
    def rollout_torch(self, actions, obs=False):
        """Rolls K open-loop action sequences out from every env's current state, H steps each, and leaves every env as it
        was (state, hints, fault bits, launch order, host mirrors, wrapper statistics).  `actions`: a contiguous float32
        tensor [K, H, num_envs, 4] on this env's device, K and H >= 1; row (k, e) starts from the state the next
        `step_torch` of env e would start from and takes `actions[k, h, e]` at its step h.  An env marked ended (NEXT_STEP
        / DISABLED, before its restart) is ended from step 0.  Returns a `Rollout` of new device tensors (`obs` only when
        `obs` is true), without host synchronisation; the hint workspace is kept on the env and grown with K."""
        self._check_started("rollout_torch")
        t, N = self.torch, self.num_envs
        if not (isinstance(actions, t.Tensor) and actions.dim() == 4 and actions.shape[0] >= 1 and actions.shape[1] >= 1):
            raise ValueError(f"actions must be a contiguous float32 tensor of shape (K, H, {N}, 4) with K, H >= 1 on {self.device}")
        K, H = actions.shape[:2]
        self._check_tensor("actions", actions, t.float32, (K, H, N, 4), contiguous=True)
        dev = self.device
        if self._rollout_hints is None or self._rollout_hints.shape[0] < K * N:
            self._rollout_hints = t.empty(K * N, NCONV, 4, dtype=t.float32, device=dev)
        reward = t.empty(K, H, N, device=dev)
        info = t.empty(K, H, N, 7, device=dev)
        flags = t.empty(K, H, N, dtype=t.uint8, device=dev)
        o = t.empty(K, H, N, 39, device=dev) if obs else None
        diag = t.empty(K, N, 2, dtype=t.int32, device=dev)
        self.engine.rollout(actions, reward, info, flags, o, diag, self._rollout_hints)
        return Rollout(reward, info, (flags & 1) != 0, (flags & 2) != 0, (flags & 4) != 0, o, diag[..., 0], diag[..., 1])

    def rollout(self, actions, obs=False):
        """`rollout_torch` from a numpy float32 array [K, H, num_envs, 4]; returns a `Rollout` of numpy arrays after one
        synchronisation.  A bad shape or dtype raises ValueError before anything runs; fault bits 1 / 2 / 4 / 8 in any row
        raise ValueError with `Engine.FAULTS`' message, as `Engine.raise_on_faults` does for `step`."""
        N = self.num_envs
        a = np.asarray(actions)
        if a.dtype != np.float32 or a.ndim != 4 or a.shape[2:] != (N, 4) or a.shape[0] < 1 or a.shape[1] < 1:
            raise ValueError(f"rollout needs actions as a float32 array of shape (K, H, {N}, 4) with K, H >= 1, got {a.dtype} {a.shape}")
        self._check_started("rollout")
        r = self.rollout_torch(self.torch.from_numpy(np.ascontiguousarray(a)).to(self.device), obs)
        host = [None if x is None else x.to("cpu", non_blocking=True) for x in r]
        if self.device.type == "cuda":
            self.torch.cuda.synchronize(self.device)
        out = Rollout(*(None if x is None else x.numpy() for x in host))
        bad = np.argwhere(out.faults & 15)
        if len(bad):
            k, e = (int(i) for i in bad[0])
            msgs = [m for b, m in Engine.FAULTS.items() if out.faults[k, e] & b]
            raise ValueError(f"rollout candidate {k}, env {e}: " + "; ".join(msgs) + f" ({len(bad)} row(s) flagged)")
        return out

    # attribute RPC used by metaworld/evaluation.py:48-169 and the reference tests
    def _current_tasks(self):
        if self._device_sampler or self._goal_bufs is not None:
            # the device chose the goals (sampler), or an episode may run on a reset_goals goal (snapshot id -1): read the
            # snapshot id of every env's running episode
            snap = self.engine.get_state()["snapshot"].astype(np.int64)
            goal = None if self._goal_bufs is None else self._goal_bufs[2].cpu().numpy()
            return [self._goal_task(e, goal[e]) if i < 0 else self._task_of_snap[int(i)] if self._device_sampler
                    else self.sub[e].current_task for e, i in enumerate(snap)]
        return [s.current_task for s in self.sub]

    def get_attr(self, name):
        if name == "terminate_on_success":
            return tuple([self.terminate_on_success] * self.num_envs)
        if name == "task_name":
            return tuple(s.task_name for s in self.sub)
        if name == "tasks":
            return tuple(s.tasks for s in self.sub)
        if name in ("_last_rand_vec", "_partially_observable"):
            key = "rand_vec" if name == "_last_rand_vec" else "partially_observable"
            return tuple(None if tk is None else tk.unpack()[key] for tk in self._current_tasks())
        if name == "max_path_length":
            return tuple([MAX_PATH_LENGTH] * self.num_envs)
        if name == "curr_path_length":
            return tuple(int(x) for x in self._ep_len)
        if name == "sample_tasks_on_reset":
            return tuple(s.sample_tasks_on_reset for s in self.sub)
        if name == "env_id":
            return tuple(s.env_id for s in self.sub)
        if name in STATE_ATTRS:
            if name != "hand_init_pos":       # a constant of the task
                self._check_started(name)
            return getattr(self._getters, name)()
        raise AttributeError(name)

    def set_attr(self, name, values):
        vals = values if isinstance(values, (list, tuple)) else [values] * self.num_envs
        if name == "terminate_on_success":
            self.call("toggle_terminate_on_success", bool(vals[0]))
        elif name == "sample_tasks_on_reset":
            for s in self.sub:
                s.rewind_pending()
            for s, v in zip(self.sub, vals):
                s.sample_tasks_on_reset = bool(v)
            if not self._needs_reset:
                self._redraw_all_pending()
        else:
            raise AttributeError(name)

    def call(self, name, *args, **kwargs):
        if name == "toggle_terminate_on_success":
            self.terminate_on_success = bool(args[0])
            self._set_engine_options()
            return tuple([None] * self.num_envs)
        if name == "toggle_sample_tasks_on_reset":
            self.set_attr("sample_tasks_on_reset", bool(args[0]))
            return tuple([None] * self.num_envs)
        if name == "sample_tasks":        # wrappers.py:121-123 / 186-188: draw a task, then reset
            for s in self.sub:
                s.rewind_pending()
                s.current_task = s.next_task()
            saved = [s.sample_tasks_on_reset for s in self.sub]
            for s in self.sub:
                s.sample_tasks_on_reset = False
            obs, info = self.reset()
            for s, v in zip(self.sub, saved):
                s.sample_tasks_on_reset = v
            self._redraw_all_pending()
            return tuple((obs[e], {}) for e in range(self.num_envs))
        if name == "get_checkpoint":
            return self.get_checkpoint()
        if name == "load_checkpoint":
            self.load_checkpoint(args[0])
            return tuple([None] * self.num_envs)
        # the reference getters and MujocoEnv / SawyerMocapBase's physics state, on every sub-env's base env
        if name in STATE_CALLS or name in ("set_state", "set_env_state", "get_env_state", "_get_obs"):
            self._check_started(name)
            return getattr(self._getters, name)(*args, **kwargs)
        return self.get_attr(name)

    # ------------------------------------------------------------------ checkpoint (metaworld/wrappers.py:125-142,190-204,275-322)
    def get_checkpoint(self, physics=True):
        """Tuple of the reference's per-sub-env ``CheckpointWrapper.get_checkpoint()`` results: ``(env_id, dict)`` with
        ``tasks`` (base64), ``rng_state`` (random select) or ``current_task_idx`` (pseudorandom), ``sample_tasks_on_reset``
        and ``env_rng_state``.  Extension (ignored by the reference's loader): ``mw_b200`` holds the env's 512-byte device
        record (qpos/qvel/warm start/mocap/frame stack/reward latches/episode counters) and the host mirrors, so a resumed
        run continues bit-identically mid-episode."""
        st = self.engine.get_state() if (physics and not self._needs_reset) else None
        goal = None if st is None or self._goal_bufs is None else self._goal_bufs[2].cpu().numpy()
        out = []
        for e, s in enumerate(self.sub):
            tasks, idx, rng_state = s._pre if s._pre is not None else (s.tasks, s.current_task_idx, s.np_random.bit_generator.state)
            ck = {"tasks": [_serialize_task(t) for t in tasks]}
            if s.pseudorandom:
                ck["current_task_idx"] = idx
            else:
                ck["rng_state"] = rng_state
            ck["sample_tasks_on_reset"] = s.sample_tasks_on_reset
            ck["env_rng_state"] = {"np_random_state": rng_state,
                                   "action_space_rng_state": s.space_rng["action_space"].bit_generator.state,
                                   "obs_space_rng_state": s.space_rng["obs_space"].bit_generator.state,
                                   "goal_space_rng_state": s.space_rng["goal_space"].bit_generator.state}
            ext = {"ep_len": int(self._ep_len[e]),
                   "current_task": None if s.current_task is None else _serialize_task(s.current_task)}
            if st is not None:
                ext["state"] = base64.b64encode(st[e].tobytes()).decode("ascii")
                if st[e]["snapshot"] < 0:        # an episode on a reset_goals goal
                    ext["goal"] = [float(x) for x in goal[e]]
            ck["mw_b200"] = ext
            out.append((s.env_id, ck))
        return tuple(out)

    def load_checkpoint(self, ckpts):
        """Accepts what the reference's ``envs.call("load_checkpoint", ckpts)`` is given: the list of ``(env_id, dict)``
        tuples; every sub-env takes the entry with its own env_id (k-th env with an id takes the k-th entry with that id:
        the ML benchmarks give every sub-env the id ``..._None``)."""
        ckpts = list(ckpts)
        used = [False] * len(ckpts)
        mine = []
        for s in self.sub:
            hit = None
            for i, (env_id, ck) in enumerate(ckpts):
                if env_id == s.env_id and not used[i]:
                    hit = i
                    break
            if hit is None:
                raise ValueError(f"Could not load checkpoint, no checkpoint found with id {s.env_id}. Checkpoint IDs: ",
                                 [env_id for env_id, _ in ckpts])
            used[hit] = True
            mine.append(ckpts[hit][1])
        new_tasks = []
        for ck in mine:
            for k in ("tasks", "sample_tasks_on_reset", "env_rng_state"):
                assert k in ck
            new_tasks += [_deserialize_task(t) for t in ck["tasks"]]
        self._ensure_snapshots(new_tasks)
        st = None
        rows, lens, cur, goals = [], [], [], {}
        for e, (s, ck) in enumerate(zip(self.sub, mine)):
            s.pending, s._pre = None, None
            s.tasks = [_deserialize_task(t) for t in ck["tasks"]]
            if s.pseudorandom:
                assert "current_task_idx" in ck
                s.current_task_idx = ck["current_task_idx"]
            else:
                assert "rng_state" in ck
            s.sample_tasks_on_reset = ck["sample_tasks_on_reset"]
            ers = ck["env_rng_state"]
            s.np_random.bit_generator.state = ers["np_random_state"] if s.pseudorandom else ck["rng_state"]
            s.space_rng["action_space"].bit_generator.state = ers["action_space_rng_state"]
            s.space_rng["obs_space"].bit_generator.state = ers["obs_space_rng_state"]
            s.space_rng["goal_space"].bit_generator.state = ers["goal_space_rng_state"]
            ext = ck.get("mw_b200")
            if ext is not None:
                rows.append(e); lens.append(ext["ep_len"])
                cur.append(None if ext["current_task"] is None else _deserialize_task(ext["current_task"]))
                if "state" in ext:
                    if st is None:
                        st = self.engine.get_state()
                    st[e] = np.frombuffer(base64.b64decode(ext["state"]), dtype=ENVSTATE_DTYPE)[0]
                    if "goal" in ext:
                        goals[e] = ext["goal"]
        self._restore_mirrors(rows, lens, cur)
        if st is not None:
            # (the ended mark: a run stopped between a terminal step and its restart)
            self._autoreset_envs.host(write=True)[rows] = st["ended"][rows] != 0
            # snapshot ids are engine-local: re-point every restored record at this engine's id for the same task
            # (an episode on a reset_goals goal keeps snapshot id -1 and takes its running goal back)
            for e, s in enumerate(self.sub):
                if s.current_task is not None and e not in goals:
                    self._ensure_snapshots([s.current_task])
                    st[e]["snapshot"] = self._snap(s.current_task)
            if goals:
                g = self._goal_buffers()[2]
                for e, v in goals.items():
                    g[e] = self.torch.tensor(v, dtype=self.torch.float64)
            self.engine.set_state(st)
            self._needs_reset = False
        if not self._needs_reset:
            for e, s in enumerate(self.sub):
                if s.current_task is None:
                    self._needs_reset = True
            if not self._needs_reset:
                for e in range(self.num_envs):
                    self._draw_pending(e)
                self._push_next()

    def close(self, **kwargs):
        if not self._closed and self._own_engine:
            self.engine.close()
        self._closed = True


def make_mt_envs(name, seed=None, num_tasks=None, num_envs=None, **kwargs):
    """``make_mt_envs`` (metaworld/__init__.py:460-513) -> MetaWorldVecEnv.  ``vector_strategy`` is accepted
    and ignored (there is one strategy: the GPU); ``autoreset_mode`` is gymnasium's (SAME_STEP by default).  For a task name the reference returns ONE wrapped env, not a vector
    (:470-478): pass ``single=True`` (what ``gym.make("Meta-World/MT1", ...)`` does) to get that object."""
    from . import benchmarks as B

    if kwargs.pop("single", False):
        from .single_env import MetaWorldSingleEnv
        kwargs.pop("autoreset_mode", None)         # one wrapped env: no vector autoreset, as in the reference (:470-478)
        return MetaWorldSingleEnv(make_mt_envs(name, seed=seed, num_tasks=num_tasks, num_envs=1, **kwargs))

    kwargs.pop("vector_strategy", None)
    bench = B.make_benchmark(name, seed, kwargs.pop("num_goals", B.N_GOALS))
    names = list(bench.train_classes)
    default = {"MT10": 10, "MT25": 25, "MT50": 50}.get(name, 1)
    tasks = [[t for t in bench.train_tasks if t.env_name == n] for n in names]
    if name in TASKS:       # MT1: _init_each_env is called without env_id (metaworld/__init__.py:471-477)
        kwargs.setdefault("checkpoint_env_ids", [None])
    return MetaWorldVecEnv(names, tasks, num_envs=num_envs, seed=seed, num_tasks=num_tasks or default, **kwargs)


def _meta_batch(bench, split, meta_batch_size, total_tasks_per_cls):
    """`_make_ml_envs_inner`'s meta-batch (metaworld/__init__.py:526-545): every class of the split gets `per` =
    meta_batch_size / (number of classes) sub-envs, the i-th of them every per-th of the class's tasks from the i-th.
    -> (env names, task lists) of the sub-envs"""
    classes = list(bench.train_classes if split == "train" else bench.test_classes)
    all_tasks = bench.train_tasks if split == "train" else bench.test_tasks
    assert meta_batch_size % len(classes) == 0, "meta_batch_size must be divisible by envs_per_task"
    per = meta_batch_size // len(classes)
    names, tasks = [], []
    for n in classes:
        ts = [t for t in all_tasks if t.env_name == n]
        if total_tasks_per_cls is not None:
            ts = ts[:total_tasks_per_cls]
        for i in range(per):
            names.append(n); tasks.append(ts[i::per])
    return names, tasks


def make_ml_envs(name, seed=None, meta_batch_size=20, total_tasks_per_cls=None, split="train", num_envs=None, **kwargs):
    """``make_ml_envs`` / ``_make_ml_envs_inner`` (metaworld/__init__.py:515-604)."""
    from . import benchmarks as B

    kwargs.pop("vector_strategy", None)
    ng = kwargs.pop("num_goals", B.N_GOALS)
    bench = B.ML1(name, seed, ng) if name in TASKS else B.make_benchmark(name, seed, ng)
    names, tasks = _meta_batch(bench, split, meta_batch_size, total_tasks_per_cls)
    kwargs.setdefault("task_select", "pseudorandom")
    kwargs.setdefault("checkpoint_env_ids", [None] * len(names))     # _init_each_env gets no env_id here (:548-560)
    return MetaWorldVecEnv(names, tasks, num_envs=num_envs, seed=seed, **kwargs)


def make_custom_mt_envs(envs_list, seed=None, use_one_hot=False, num_envs=None, **kwargs):
    """``Meta-World/custom-mt-envs`` (metaworld/__init__.py:741-783): sub-env i is ``make_mt_envs(envs_list[i],
    num_tasks=len(envs_list), env_id=i, seed=seed + i)``, i.e. an MT1 benchmark of its own with its own seed."""
    from . import benchmarks as B

    kwargs.pop("vector_strategy", None)
    ng = kwargs.pop("num_goals", B.N_GOALS)
    seeds = [None if not seed else seed + i for i in range(len(envs_list))]
    tasks = [B.MT1(n, sd, ng).train_tasks for n, sd in zip(envs_list, seeds)]
    return MetaWorldVecEnv(list(envs_list), tasks, num_envs=num_envs, seed=seed, use_one_hot=use_one_hot, num_tasks=len(envs_list),
                           type_seeds=seeds, **kwargs)


def make_custom_ml_envs(train_envs, test_envs, seed=None, meta_batch_size=20, total_tasks_per_cls=None, split="train", num_envs=None, **kwargs):
    """``Meta-World/custom-ml-envs`` (metaworld/__init__.py:370-395,785-820): ``CustomML`` + ``_make_ml_envs_inner``."""
    from . import benchmarks as B

    if set(train_envs) & set(test_envs):
        raise ValueError("The test tasks cannot contain any of the train tasks.")
    kwargs.pop("vector_strategy", None)
    bench = B.Benchmark(train_envs, test_envs, True, seed, n_goals=kwargs.pop("num_goals", B.N_GOALS))
    names, tasks = _meta_batch(bench, split, meta_batch_size, total_tasks_per_cls)
    # _make_ml_envs_inner is reached without the pseudorandom partial here: _init_each_env's default task_select="random"
    kwargs.setdefault("checkpoint_env_ids", [None] * len(names))
    return MetaWorldVecEnv(names, tasks, num_envs=num_envs, seed=seed, **kwargs)
