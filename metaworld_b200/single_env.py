"""Single-environment surface of the reference over the CUDA engine.

Two classes:

* ``SawyerXYZEnvB200`` -- what ``mt1.train_classes[name]()`` gives in the reference: the bare ``SawyerXYZEnv`` protocol
  (metaworld/sawyer_xyz_env.py:143-719): ``set_task`` / ``reset`` / ``step`` / ``evaluate_state`` / ``compute_reward`` /
  ``seed`` and the attributes the reference's tests read (``_partially_observable``, ``_last_rand_vec``, ``_target_pos``,
  ``obj_init_pos``, ``task_name``, ``max_path_length``, ``curr_path_length``, ``observation_space``, ``action_space``,
  ``np_random``), with the same errors (RuntimeError before ``set_task``, ValueError when stepping past the horizon,
  AssertionError on a wrong action length).  One engine with one environment; every call is a kernel launch through the
  C ABI -- there is no CPU path.
* ``MetaWorldSingleEnv`` -- what ``gym.make("Meta-World/MT1", env_name=...)`` / ``make_mt_envs(<task name>)`` gives: the
  same env under the wrapper stack of ``_init_each_env`` (metaworld/__init__.py:398-458: TimeLimit, terminate-on-success,
  one-hot, episode statistics, random task selection on reset, checkpoint).  It is a 1-env ``MetaWorldVecEnv`` with the
  batch dimension removed and WITHOUT autoreset, like the reference's non-vector env.

A single environment uses one warp of one SM: this surface exists so that the reference's single-env tests and user code
can be pointed at the engine unchanged, not for throughput.
"""
from __future__ import annotations

import numpy as np

from . import _gym
from .benchmarks import REFERENCE_CLASS, Task
from .engine import INFO_KEYS, Engine
from .getters import STATE_CALLS, StateGetters
from .tasks import TASKS
from .vector_env import MAX_PATH_LENGTH, MetaWorldVecEnv

_HAND_LOW = np.array([-0.525, 0.348, -0.0525])     # SawyerXYZEnv._HAND_SPACE (sawyer_xyz_env.py:146-150)
_HAND_HIGH = np.array([+0.525, 1.025, 0.7])


def _assert_task_is_set(fn):          # SawyerXYZEnv._Decorators.assert_task_is_set (sawyer_xyz_env.py:159-173)
    def inner(self, *a, **k):
        if not self._set_task_called:
            raise RuntimeError("You must call env.set_task before using env." + fn.__name__)
        return fn(self, *a, **k)
    inner.__name__ = fn.__name__
    return inner


class SawyerXYZEnvB200:
    max_path_length = MAX_PATH_LENGTH
    TARGET_RADIUS = 0.05
    metadata = {"render_modes": [], "render_fps": 80}

    def __init__(self, env_name, render_mode=None, reward_function_version=None, device=0, engine=None, **unused):
        if env_name not in TASKS:
            raise ValueError(f"{env_name} is not a V3 environment")
        if render_mode is not None:
            raise NotImplementedError("rendering is outside the hot path this package replaces")
        if reward_function_version not in (None, "v2"):
            raise NotImplementedError("only the default v2 rewards are implemented on the device")
        self.env_name = env_name
        self.spec_ = TASKS[env_name]
        self.task_name = REFERENCE_CLASS[env_name].rsplit(".", 1)[1]      # self.__class__.__name__ in the reference (:252)
        self.engine = engine or Engine([env_name], device=device)
        self._own_engine = engine is None
        self.torch = self.engine.torch
        self.engine.set_envs([0])
        # no wrapper here: the horizon check is SawyerXYZEnv's own (max_path_length), success never terminates
        self.engine.set_options(MAX_PATH_LENGTH, False, 0)
        # autoreset off (the horizon is SawyerXYZEnv's own): at truncation the env keeps its terminal state, which the
        # state getters read, until reset().  This also applies to an engine passed in through `engine=`.
        self.engine.set_autoreset_mode("Disabled")
        self._getters = StateGetters(self.engine, [env_name], check_ready=self._check_reset)
        self.curr_path_length = 0
        self._goal_site_written = False
        self._partially_observable = True            # until set_task (sawyer_xyz_env.py:208)
        self._set_task_called = False
        self._last_rand_vec = None
        self._freeze_rand_vec = True
        self.seeded_rand_vec = False                 # unfrozen draws from self.np_random instead of np.random (:702-710)
        self._snap_cache: dict = {}
        self._snap_id = None
        self._did_reset = False
        self.np_random = np.random.default_rng()
        self.action_space = _gym.Box(-np.ones(4, np.float32), np.ones(4, np.float32), dtype=np.float32)
        self.goal_low, self.goal_high = np.array(self.spec_.goal_low, dtype=np.float64), np.array(self.spec_.goal_high, dtype=np.float64)
        self.goal_space = _gym.Box(self.goal_low, self.goal_high, dtype=np.float64)
        self.hand_init_pos = np.array(self.spec_.hand_init_pos, dtype=np.float64)
        dev = self.engine.device
        t = self.torch
        self.d_obs = t.zeros(1, 39, device=dev); self.d_rew = t.zeros(1, device=dev)
        self.d_term = t.zeros(1, dtype=t.uint8, device=dev); self.d_trunc = t.zeros(1, dtype=t.uint8, device=dev)
        self.d_info = t.zeros(1, 9, device=dev); self.d_fobs = t.zeros(1, 39, device=dev); self.d_finfo = t.zeros(1, 8, device=dev)
        self.d_act = t.zeros(1, 4, device=dev); self.d_sid = t.zeros(1, dtype=t.int32, device=dev)
        self._goal_bufs = None       # (goal row, goal vectors, observability, mask) of the unfrozen reset, made on first use
        self._last_stable_obs = None

    # ---- spaces (sawyer_xyz_env.py:529-577): recomputed when observability changes, like the cached_property there
    @property
    def observation_space(self):
        inf = np.full(14, np.inf)
        gl, gh = (np.zeros(3), np.zeros(3)) if self._partially_observable else (self.goal_low, self.goal_high)
        return _gym.Box(np.hstack((_HAND_LOW, -1.0, -inf, _HAND_LOW, -1.0, -inf, gl)),
                        np.hstack((_HAND_HIGH, 1.0, inf, _HAND_HIGH, 1.0, inf, gh)), dtype=np.float64)

    sawyer_observation_space = observation_space

    def seed(self, seed):
        assert seed is not None
        self.np_random = np.random.Generator(np.random.PCG64(seed))
        self.action_space.seed(seed)
        self.goal_space.seed(seed)
        return [seed]

    def set_task(self, task: Task):
        """sawyer_xyz_env.py:298-318."""
        self._set_task_called = True
        data = task.unpack()
        cls = data["env_cls"]
        cls_name = cls if isinstance(cls, str) else f"{cls.__module__}.{cls.__name__}"
        assert cls_name in (REFERENCE_CLASS[self.env_name], self.env_name), "task belongs to another environment class"
        self._freeze_rand_vec = True
        self._last_rand_vec = np.asarray(data["rand_vec"], dtype=np.float64)
        self._partially_observable = bool(data["partially_observable"])

    def _snapshot(self, pass1=None):
        key = (self._last_rand_vec.tobytes(), self._partially_observable, None if pass1 is None else np.asarray(pass1).tobytes())
        if key not in self._snap_cache:
            rv = np.zeros((1, 6)); rv[0, : len(self._last_rand_vec)] = self._last_rand_vec
            rv1 = None
            if pass1 is not None:
                rv1 = np.zeros((1, 6)); rv1[0, : len(pass1)] = pass1
            self._snap_cache[key] = int(self.engine.build_snapshots([0], rv, [self._partially_observable], rand_vec_pass1=rv1)[0])
        return self._snap_cache[key]

    def reset(self, seed=None, options=None, _pass1=None):
        """sawyer_xyz_env.py:664-682 (`seed` / `options` ignored there too).  The double-pass reset is evaluated by the
        device once per distinct (rand_vec, observability) and cached as an episode-start snapshot.  With
        `_freeze_rand_vec` False each reset_model pass draws a new goal as `_get_state_rand_vec` does (:697-719), from
        np.random or, when `seeded_rand_vec`, from `np_random`; `_last_rand_vec` is the second pass's, and the episode
        starts from a goal row built on the device, which the snapshot table never holds."""
        self.curr_path_length = 0
        if not self._freeze_rand_vec:
            self._reset_unfrozen()
        else:
            assert self._last_rand_vec is not None, "set_task must be called before reset (the reference asserts in _get_state_rand_vec)"
            self._snap_id = self._snapshot(_pass1)
            self.d_sid[0] = self._snap_id
            self.engine.reset(self.d_sid, self.d_obs)
        self._did_reset = True
        self._goal_site_written = self.env_name == "shelf-place-v3"
        return self.d_obs[0].cpu().numpy().astype(np.float64), {}

    def _reset_unfrozen(self):
        from .benchmarks import draw_rand_vec

        src = self.np_random if self.seeded_rand_vec else np.random
        first = draw_rand_vec(self.spec_, src)                 # reset_model pass 1
        self._last_rand_vec = draw_rand_vec(self.spec_, src)   # pass 2
        t, dev = self.torch, self.engine.device
        if self._goal_bufs is None:
            self._goal_bufs = (t.zeros(1, 768, dtype=t.uint8, device=dev), t.zeros(2, 1, 6, dtype=t.float64, device=dev),
                               t.zeros(1, dtype=t.uint8, device=dev), t.ones(1, dtype=t.bool, device=dev))
        row, rv, po, mask = self._goal_bufs
        v = np.zeros((2, 1, 6))
        v[0, 0, : first.size], v[1, 0, : self._last_rand_vec.size] = first, self._last_rand_vec
        rv.copy_(t.from_numpy(v))
        po.fill_(int(self._partially_observable))
        self.engine.build_goal_rows(mask, rv[1], rv[0], po, row)
        self.engine.reset_rows(mask, row, self.d_obs)

    @_assert_task_is_set
    def step(self, action):
        """sawyer_xyz_env.py:580-642."""
        assert len(action) == 4, f"Actions should be size 4, got {len(action)}"
        if self.curr_path_length >= self.max_path_length:
            raise ValueError("You must reset the env manually once truncate==True")
        if not self._did_reset:
            raise RuntimeError("reset() must be called before step() (the device state is created by reset)")
        self.d_act[0] = self.torch.as_tensor(np.asarray(action, dtype=np.float32))
        self.engine.step(self.d_act, self.d_obs, self.d_rew, self.d_term, self.d_trunc, self.d_info, self.d_fobs, self.d_finfo, self.d_sid)
        self.curr_path_length += 1
        self._goal_site_written = False
        rec = self.d_info[0].cpu().numpy()
        truncate = self.curr_path_length == self.max_path_length
        # autoreset is off: at the horizon the env keeps its terminal state (the state getters read it) until reset()
        obs = self.d_obs[0].cpu().numpy().astype(np.float64)
        self._last_stable_obs = obs
        info = {k: float(rec[i]) for i, k in enumerate(INFO_KEYS)}
        return obs, float(rec[7]), False, truncate, info

    @_assert_task_is_set
    def evaluate_state(self, obs, action):
        """Reward and info of the CURRENT physics state for the given (obs, action) (sawyer_xyz_env.py:644-656 + the task's
        evaluate_state): one forward pass + the task's reward code on the device, no state change."""
        o = self.torch.as_tensor(np.asarray(obs, dtype=np.float32).reshape(1, 39)).to(self.engine.device)
        a = self.torch.as_tensor(np.asarray(action, dtype=np.float32).reshape(1, 4)).to(self.engine.device)
        out = self.torch.zeros(1, 8, device=self.engine.device)
        self.engine.evaluate(a, o, out)
        r = out[0].cpu().numpy()
        return float(r[7]), {k: float(r[i]) for i, k in enumerate(INFO_KEYS)}

    @_assert_task_is_set
    def compute_reward(self, action, obs):
        """The reference returns a task-specific tuple whose first element is the reward and whose other elements are the
        quantities its ``evaluate_state`` puts into ``info``.  Here: ``(reward, obj_to_target, grasp_reward,
        in_place_reward)`` for every task (documented deviation: the reference's per-task tuple layouts differ)."""
        r, info = self.evaluate_state(obs, action)
        return r, info["obj_to_target"], info["grasp_reward"], info["in_place_reward"]

    # ---- state getters (sawyer_xyz_env.py:67-107, 363-473, 513-535; MujocoEnv.set_state / get_body_com): row 0 of the
    # shared implementation, which runs `_check_reset` before it queries, observes or writes the device state
    def _check_reset(self):
        if not self._did_reset:
            raise RuntimeError("reset() must be called before reading or setting the state (the device state is created by reset)")

    @property
    def _target_pos(self):
        return self._getters._target_pos()[0]

    @property
    def obj_init_pos(self):
        return self._getters.obj_init_pos()[0]

    def get_env_state(self):
        return self._getters.get_env_state()[0]

    def set_state(self, qpos, qvel):
        """MujocoEnv.set_state (gymnasium mujoco_env.py), with its shape assertion.  qvel is stored as float32; the frame
        stack, mocap and task state are kept, and the observation of the new state is what `_get_obs()` returns."""
        self._getters.set_state(qpos, qvel)
        self._goal_site_written = False      # MujocoEnv.set_state runs mj_forward

    def set_env_state(self, state):
        """SawyerMocapBase.set_env_state((qpos, qvel)) (sawyer_xyz_env.py:97-107)."""
        qpos, qvel = state
        self.set_state(qpos, qvel)

    def _get_obs(self):
        return self._getters._get_obs()[0]

    def get_endeff_pos(self):
        return self._getters.get_endeff_pos()[0]

    @property
    def tcp_center(self):
        return self._getters.tcp_center()[0]

    def _get_pos_objects(self):
        return self._getters._get_pos_objects()[0]

    def _get_quat_objects(self):
        return self._getters._get_quat_objects()[0]

    def _get_pos_goal(self):
        return self._getters._get_pos_goal()[0]

    def _get_obs_dict(self):
        return self._getters._get_obs_dict()[0]

    def _get_site_pos(self, site_name):
        if site_name == "goal" and self._goal_site_written:
            return self._target_pos        # reset_model's _set_pos_site("goal", ...) holds until the next forward pass
        return self._getters._get_site_pos(site_name)[0]

    def get_body_com(self, body_name):
        return self._getters.get_body_com(body_name)[0]

    def _get_id_main_object(self):
        return self._getters._get_id_main_object()[0]

    def touching_object(self, object_geom_id):
        return self._getters.touching_object(object_geom_id)[0]

    @property
    def touching_main_object(self):
        return self._getters.touching_main_object()[0]

    @property
    def init_tcp(self):
        return self._getters.init_tcp()[0]

    @property
    def init_left_pad(self):
        return self._getters.init_left_pad()[0]

    @property
    def init_right_pad(self):
        return self._getters.init_right_pad()[0]

    def close(self):
        if self._own_engine and self.engine is not None:
            self.engine.close()
        self.engine = None


class MetaWorldSingleEnv:
    """``make_mt_envs("<task>-v3", ...)`` / ``gym.make("Meta-World/MT1", env_name=...)``: the wrapped single env."""

    metadata = {"render_modes": []}

    def __init__(self, vec: MetaWorldVecEnv):
        assert vec.num_envs == 1
        self.vec = vec
        self.observation_space = vec.single_observation_space
        self.action_space = vec.single_action_space
        self._over = False           # the last step ended the episode (the kernel has already restarted it: SAME_STEP)

    @property
    def unwrapped(self):
        return self

    def reset(self, *, seed=None, options=None):
        if self._over:
            # the autoreset inside the terminal step already drew the task the reference's reset() would draw now and
            # started its episode: hand out that observation instead of drawing again
            self._over = False
            # what the vector step returned for the restarted episode (the optional per-env wrappers already saw this reset)
            return self._restart_obs[0], {}
        obs, info = self.vec.reset(seed=seed, options=options)
        return obs[0], info

    def step(self, action):
        if self._over:
            raise ValueError("You must reset the env manually once truncate==True")
        obs, r, term, trunc, infos = self.vec.step(np.asarray(action, dtype=np.float32)[None])
        if term[0] or trunc[0]:
            self._over = True
            self._restart_obs = np.array(obs)
            fi = infos["final_info"]
            info = {k: float(fi[k][0]) for k in INFO_KEYS}
            info["episode"] = {k: fi["episode"][k][0] for k in ("r", "l", "t")}
            return infos["final_obs"][0], float(r[0]), bool(term[0]), bool(trunc[0]), info
        return obs[0], float(r[0]), False, False, {k: float(infos[k][0]) for k in INFO_KEYS}

    # the attribute / method names reached through env.unwrapped / get_wrapper_attr in the reference
    def __getattr__(self, name):
        if name in ("toggle_terminate_on_success", "toggle_sample_tasks_on_reset", "sample_tasks", "get_checkpoint",
                    "load_checkpoint") + STATE_CALLS:
            def call(*a, **k):
                out = self.vec.call(name, *a, **k)
                return out[0] if isinstance(out, tuple) and len(out) == 1 else out
            return call
        try:
            return self.vec.get_attr(name)[0]
        except AttributeError:
            raise AttributeError(name) from None

    def get_wrapper_attr(self, name):
        return getattr(self, name)

    def close(self):
        self.vec.close()


def make_goal_env(env_name, seed=None, observable=False, **kwargs):
    """``Meta-World/goal_hidden`` / ``goal_observable`` (metaworld/env_dict.py:130-212, metaworld/__init__.py:686-705): a bare
    env whose single goal is drawn at construction -- ``np.random.seed(seed)``, one ``reset()`` with an unfrozen rand_vec
    (two ``reset_model`` passes = two draws, the second is kept) -- and then frozen."""
    from .benchmarks import draw_rand_vec

    for suffix in ("-goal-hidden", "-goal-observable"):
        env_name = env_name.replace(suffix, "")
    env = SawyerXYZEnvB200(env_name, **kwargs)
    rs = np.random.RandomState(seed) if seed is not None else np.random.RandomState()
    first = draw_rand_vec(env.spec_, rs)             # reset_model pass 1 (its traces survive in the construction-time state)
    env._last_rand_vec = draw_rand_vec(env.spec_, rs)
    env._partially_observable = not observable
    env._set_task_called = True
    env.reset(_pass1=first)
    if seed is not None:
        env.seed(seed)
    return env
