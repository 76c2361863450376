"""ctypes binding of libmwb200.so (C ABI: include/metaworld_b200.h) over torch CUDA tensors.

torch is only plumbing here: it owns device buffers and streams; all computation happens inside the
CUDA library.  There is no CPU fallback: constructing an `Engine` without the built library or without a
CUDA device raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import lower, modelzoo
from .tasks import MOVED_SITES, TARGET_ALIAS, TASKS, TaskSpec

_LIB = None
_LIB64 = None
_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("MW_B200_LIB") or os.path.join(_HERE, "libmwb200.so")   # MW_B200_LIB=.../libmwb200_f64.so selects the double build
SO64_PATH = os.path.join(_HERE, "libmwb200_f64.so")   # same kernels with real=double: builds the episode-start snapshots

TASKCONST_DTYPE = np.dtype([("task_id", "i4"), ("nframe_task", "i4"), ("main_geom", "i4"), ("pad", "i4"),
                            ("hand_init", "f4", 3), ("mocap_lo", "f4", 3), ("mocap_hi", "f4", 3),
                            ("goal_lo", "f4", 3), ("goal_hi", "f4", 3), ("movable_pos0", "f4", 3), ("p", "f4", 16)])
ENVSTATE_DTYPE = np.dtype([("qpos", "f8", 18), ("qvel", "f4", 17), ("warm", "f4", 17), ("mocap_pos", "f4", 3),
                           ("prev_obs", "f4", 18), ("shift", "f4", 3), ("target", "f4", 3), ("obj_init", "f4", 3),
                           ("init_tcp", "f4", 3), ("scal", "f4", 16), ("path_len", "f4"),
                           ("partially_observable", "f4"), ("snapshot", "f4"), ("episode", "f4"), ("ep_return", "f4"),
                           ("ended", "f4"), ("gripper_ctrl", "f4"), ("pad", "f4", 2)])
SNAPSHOT_DTYPE = np.dtype([("st", ENVSTATE_DTYPE), ("obs", "f4", 39), ("pad", "f4", 25)])
MAXNQ, MAXDOF = 18, 17      # the padded qpos / qvel layout of set_physics / get_physics (ENVSTATE_DTYPE's qpos / qvel)
INFO_KEYS = ["success", "near_object", "grasp_success", "grasp_reward", "in_place_reward", "obj_to_target",
             "unscaled_reward"]


class EngineError(RuntimeError):
    pass


def _load(path):
    if not os.path.exists(path):
        raise EngineError(f"{path} is missing: build it with `python -m metaworld_b200.build` (and `--double`); "
                          "the engine has no CPU fallback")
    L = C.CDLL(path)
    L.mw_last_error.restype = C.c_char_p
    L.mw_build_info.restype = C.c_char_p
    vp, ip = C.c_void_p, C.c_int
    L.mw_create.argtypes = [C.POINTER(vp), ip, ip, vp, vp, C.POINTER(vp), vp]
    L.mw_destroy.argtypes = [vp]
    L.mw_set_envs.argtypes = [vp, ip, vp]
    L.mw_build_snapshots.argtypes = [vp, ip, vp, vp, vp, vp, vp]
    L.mw_append_snapshots.argtypes = [vp, ip, vp, vp]
    L.mw_num_snapshots.argtypes = [vp]
    L.mw_get_snapshots.argtypes = [vp, ip, ip, vp]
    L.mw_reset.argtypes = [vp, ip, vp, vp, vp, ip, vp]
    L.mw_step.argtypes = [vp, vp, vp, ip, vp, vp, vp, vp, ip, vp, vp, vp, vp]
    L.mw_set_autoreset_mode.argtypes = [vp, ip]
    L.mw_reset_masked.argtypes = [vp, vp, vp, vp, ip, vp]
    L.mw_set_options.argtypes = [vp, ip, ip, C.c_ulonglong]
    L.mw_set_goal_sets.argtypes = [vp, vp, vp]
    L.mw_get_state.argtypes = [vp, vp]
    L.mw_set_state.argtypes = [vp, vp]
    L.mw_debug_substeps.argtypes = [vp, ip, vp, vp]
    L.mw_get_counters.argtypes = [vp, vp]
    L.mw_debug_forward.argtypes = [vp, vp, vp, vp]
    L.mw_get_profile.argtypes = [vp, vp]
    L.mw_rebalance.argtypes = [vp]
    L.mw_get_env_cost.argtypes = [vp, vp]
    L.mw_evaluate.argtypes = [vp, vp, vp, ip, vp, vp]
    L.mw_set_physics.argtypes = [vp, vp, vp, vp, vp]
    L.mw_get_physics.argtypes = [vp, vp, vp, vp]
    L.mw_observe.argtypes = [vp, vp, vp, ip, vp]
    L.mw_expert_actions.argtypes = [vp, vp, ip, ip, vp, vp]
    L.mw_query.argtypes = [vp, vp, vp, vp, ip, vp, vp, vp, vp]
    L.mw_get_faults.argtypes = [vp, vp]
    L.mw_set_profiling.argtypes = [vp, ip]
    L.mw_get_env_profile.argtypes = [vp, vp]
    assert L.mw_sizeof_model() == lower.DTYPE.itemsize, "MwModel layout mismatch (rebuild the library)"
    assert L.mw_sizeof_taskconst() == TASKCONST_DTYPE.itemsize
    assert L.mw_sizeof_envstate() == ENVSTATE_DTYPE.itemsize == 512
    assert L.mw_sizeof_snapshot() == SNAPSHOT_DTYPE.itemsize == 768
    return L


def lib():
    global _LIB
    if _LIB is None:
        _LIB = _load(SO_PATH)
    return _LIB


def lib64():
    """The float64 build of the same CUDA kernels.  Episode-start snapshots (the reference's 2 x 250-substep reset) are
    computed with it once per goal, so that contact-rich resting configurations start from the float64 answer."""
    global _LIB64
    if _LIB64 is None:
        _LIB64 = _load(SO64_PATH)
    return _LIB64


def _ck(rc, L=None):
    if rc != 0:
        raise EngineError((L or lib()).mw_last_error().decode() or f"libmwb200 error {rc}")


def expert_actions(task_ids, obs, out):
    """metaworld.policies on the device (mw_expert_actions): `out[i]` = the scripted expert action of task `task_ids[i]`
    (metaworld_b200.tasks.TASK_IDS) for observation row `obs[i, :39]`, unclipped; an unknown id gives a NaN row.  CUDA
    tensors on one device: `task_ids` int32 [n] contiguous, `obs` float32 [n, >= 39] with contiguous rows, `out` float32
    [n, 4] contiguous.  Asynchronous on the current stream; needs no Engine."""
    import torch
    n = task_ids.shape[0] if task_ids.dim() == 1 else -1
    ok = (n >= 0 and task_ids.dtype == torch.int32 and task_ids.is_contiguous() and obs.dtype == torch.float32
          and obs.dim() == 2 and obs.shape[0] == n and obs.shape[1] >= 39 and obs.stride(1) == 1
          and out.dtype == torch.float32 and tuple(out.shape) == (n, 4) and out.is_contiguous()
          and task_ids.is_cuda and obs.device == task_ids.device == out.device)
    if not ok:
        raise ValueError("expert_actions needs task_ids int32 [n], obs float32 [n, >= 39] (unit column stride) and out "
                         "float32 [n, 4], contiguous, on one CUDA device")
    with torch.cuda.device(obs.device):
        stream = C.c_void_p(torch.cuda.current_stream(obs.device).cuda_stream)
        _ck(lib().mw_expert_actions(C.c_void_p(task_ids.data_ptr()), C.c_void_p(obs.data_ptr()), obs.stride(0), n,
                                    C.c_void_p(out.data_ptr()), stream))
    return out


_LOWERED: dict = {}


def lowered(spec: TaskSpec) -> lower.Lowered:
    if spec.name not in _LOWERED:
        m = modelzoo.full_model(spec.xml)
        _LOWERED[spec.name] = lower.lower(m, spec.movable, spec.frames)
    return _LOWERED[spec.name]


def task_const(spec: TaskSpec, lw: lower.Lowered) -> np.ndarray:
    tc = np.zeros((), dtype=TASKCONST_DTYPE)
    tc["task_id"] = spec.task_id
    tc["nframe_task"] = len(spec.frames)
    tc["main_geom"] = lw.geom_names.index(spec.main_geom) if spec.main_geom in lw.geom_names else -1
    tc["hand_init"] = spec.hand_init_pos
    tc["mocap_lo"], tc["mocap_hi"] = spec.hand_low, spec.hand_high
    tc["goal_lo"], tc["goal_hi"] = spec.goal_low, spec.goal_high
    if spec.movable:
        m = modelzoo.full_model(spec.xml)
        tc["movable_pos0"] = m.arrays["body_pos"][m.names["body"].index(spec.movable)]
    p = np.zeros(16, dtype=np.float32)
    p[: len(spec.params)] = spec.params
    if spec.site_params:
        mm = modelzoo.full_model(spec.xml)
        for k, nm in enumerate(spec.site_params):
            p[3 * k: 3 * k + 3] = mm.arrays["site_pos"][mm.names["site"].index(nm)]
    # collider slots of the two finger pads (touching_object, sawyer_xyz_env.py:401-440)
    p[14] = lw.geom_names.index("leftpad_geom")
    p[15] = lw.geom_names.index("rightpad_geom")
    tc["p"] = p
    return tc


class Engine:
    """One engine per process / GPU.  `task_names[i]` defines model slot i."""

    def __init__(self, task_names, device=0):
        import torch

        if not torch.cuda.is_available():
            raise EngineError("CUDA device required: metaworld_b200 has no CPU execution path")
        self.torch = torch
        self.device = torch.device("cuda", device)
        self.specs = [TASKS[n] for n in task_names]
        self.lowered = [lowered(s) for s in self.specs]
        models = np.stack([lw.rec for lw in self.lowered])
        tcs = np.stack([task_const(s, lw) for s, lw in zip(self.specs, self.lowered)])
        self._mesh = [np.ascontiguousarray(lw.meshvert, dtype=np.float32) for lw in self.lowered]
        ptrs = (C.c_void_p * len(self._mesh))(*[m.ctypes.data if len(m) else None for m in self._mesh])
        nmv = np.array([len(m) for m in self._mesh], dtype=np.int32)
        self.h = C.c_void_p()
        self._create_args = (device, len(self.specs), models, tcs, ptrs, nmv)
        _ck(lib().mw_create(C.byref(self.h), device, len(self.specs), models.ctypes.data, tcs.ctypes.data, ptrs,
                            nmv.ctypes.data))
        self.h64 = None
        self.n_envs = 0
        self._query_tables = {}      # device copies of the mw_query tables, by frame list / geom list

    def close(self):
        if getattr(self, "h64", None):
            lib64().mw_destroy(self.h64)
            self.h64 = None
        if getattr(self, "h", None):
            lib().mw_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_envs(self, env_model):
        em = np.ascontiguousarray(env_model, dtype=np.int32)
        _ck(lib().mw_set_envs(self.h, len(em), em.ctypes.data))
        self.n_envs = len(em)
        self.env_model = em

    def set_options(self, max_episode_steps=500, terminate_on_success=False, seed=0):
        _ck(lib().mw_set_options(self.h, int(max_episode_steps), int(bool(terminate_on_success)), int(seed) & (2**64 - 1)))

    def build_snapshots(self, model_idx, rand_vec, partially_observable, precise=None, rand_vec_pass1=None):
        """Episode-start snapshots for (model slot, rand_vec) pairs.  `precise` (default: on unless
        MW_B200_SNAPSHOT_F32=1) runs the reset on the float64 build of the kernels and uploads the records.
        `rand_vec_pass1`: the vector of the first reset_model pass when it differs (unfrozen rand_vec, see the header)."""
        mi = np.ascontiguousarray(model_idx, dtype=np.int32)

        def pack(v):
            out = np.zeros((len(mi), 6), dtype=np.float64)     # the goal vector stays float64 from Task.data to the device
            v = np.asarray(v, dtype=np.float64).reshape(len(mi), -1)
            out[:, : v.shape[1]] = v
            return out

        rv = pack(rand_vec)
        rv1 = None if rand_vec_pass1 is None else pack(rand_vec_pass1)
        p1 = None if rv1 is None else rv1.ctypes.data
        po = np.ascontiguousarray(partially_observable, dtype=np.uint8)
        ids = np.zeros(len(mi), dtype=np.int32)
        if precise is None:
            precise = os.environ.get("MW_B200_SNAPSHOT_F32", "0") != "1" and SO_PATH != SO64_PATH
        if not precise:
            _ck(lib().mw_build_snapshots(self.h, len(mi), mi.ctypes.data, rv.ctypes.data, p1, po.ctypes.data, ids.ctypes.data))
            return ids
        L = lib64()
        if self.h64 is None:
            device, nm, models, tcs, ptrs, nmv = self._create_args
            self.h64 = C.c_void_p()
            _ck(L.mw_create(C.byref(self.h64), device, nm, models.ctypes.data, tcs.ctypes.data, ptrs, nmv.ctypes.data), L)
        first = L.mw_num_snapshots(self.h64)
        _ck(L.mw_build_snapshots(self.h64, len(mi), mi.ctypes.data, rv.ctypes.data, p1, po.ctypes.data, None), L)
        rec = np.zeros(len(mi), dtype=SNAPSHOT_DTYPE)
        _ck(L.mw_get_snapshots(self.h64, first, len(mi), rec.ctypes.data), L)
        _ck(lib().mw_append_snapshots(self.h, len(mi), rec.ctypes.data, ids.ctypes.data))
        return ids

    def get_snapshots(self, first=0, n=None):
        n = lib().mw_num_snapshots(self.h) - first if n is None else n
        out = np.zeros(n, dtype=SNAPSHOT_DTYPE)
        _ck(lib().mw_get_snapshots(self.h, first, n, out.ctypes.data))
        return out

    def set_goal_sets(self, first, count):
        f = np.ascontiguousarray(first, dtype=np.int32)
        c = np.ascontiguousarray(count, dtype=np.int32)
        _ck(lib().mw_set_goal_sets(self.h, f.ctypes.data, c.ctypes.data))

    @staticmethod
    def _p(t):
        return None if t is None else C.c_void_p(t.data_ptr())

    def _stream(self):
        return C.c_void_p(self.torch.cuda.current_stream(self.device).cuda_stream)

    def reset(self, snapshot_ids, obs, env_ids=None):
        n = snapshot_ids.numel()
        _ck(lib().mw_reset(self.h, n, self._p(env_ids), self._p(snapshot_ids), self._p(obs), obs.stride(0), self._stream()))

    def step(self, actions, obs, reward, terminated, truncated, info, final_obs=None, final_info=None, next_snapshot=None):
        _ck(lib().mw_step(self.h, self._p(actions), self._p(obs), obs.stride(0), self._p(reward), self._p(terminated),
                          self._p(truncated), self._p(info), info.stride(0), self._p(final_obs), self._p(final_info),
                          self._p(next_snapshot), self._stream()))

    AUTORESET_MODES = {"SameStep": 0, "NextStep": 1, "Disabled": 2}     # gymnasium.vector.AutoresetMode values -> MW_AUTORESET_*

    def set_autoreset_mode(self, mode):
        """`mode`: "SameStep" | "NextStep" | "Disabled" (mw_set_autoreset_mode); applies from the next `step`."""
        _ck(lib().mw_set_autoreset_mode(self.h, self.AUTORESET_MODES.get(mode, -1)))

    def reset_masked(self, mask, obs, snapshot_ids=None):
        """Restarts the envs with `mask` set (uint8/bool device tensor [n_envs]) from `snapshot_ids` (int32 device tensor
        [n_envs], read at the masked rows) or, when None, from the device sampler's draw; writes those rows of `obs`."""
        _ck(lib().mw_reset_masked(self.h, self._p(mask), self._p(snapshot_ids), self._p(obs), obs.stride(0), self._stream()))

    def evaluate(self, actions, obs, out):
        """evaluate_state for every env's current state: out [n, 8] = info[7], reward (mw_evaluate)."""
        _ck(lib().mw_evaluate(self.h, self._p(actions), self._p(obs), obs.stride(0), self._p(out), self._stream()))

    def set_physics(self, mask, qpos, qvel):
        """MujocoEnv.set_state for the envs with `mask` set (bool/uint8 device tensor [n_envs]): `qpos` float64 [n_envs, 18],
        `qvel` float64 [n_envs, 17] (contiguous device tensors; columns past each model's nq / nv are ignored, qvel is
        rounded to float32).  Changes nothing else of the state (mw_set_physics)."""
        _ck(lib().mw_set_physics(self.h, self._p(mask), self._p(qpos), self._p(qvel), self._stream()))

    def get_physics(self, qpos, qvel):
        """Writes every env's qpos into `qpos` (float64 device tensor [n_envs, 18]) and qvel into `qvel` ([n_envs, 17]);
        columns past nq / nv are zero (mw_get_physics)."""
        _ck(lib().mw_get_physics(self.h, self._p(qpos), self._p(qvel), self._stream()))

    def observe(self, mask, obs):
        """_get_obs() of the current state for the envs with `mask` set, into the first 39 columns of their rows of `obs`
        (float32 device tensor [n_envs, >= 39]); commits their frame stack (mw_observe)."""
        _ck(lib().mw_observe(self.h, self._p(mask), self._p(obs), obs.stride(0), self._stream()))

    def query(self, mask, frame=None, pose=None, frames=None, touching=None, main_geom=None):
        """Read-only accessors of the current state for the envs with `mask` set (mw_query), into the given device tensors;
        each output may be None.  `frame` float32 [n_envs, 18]: columns 0..17 of the next `observe`, without committing
        the frame stack.  `pose` float64 [n_envs, K, 7] (xpos, quat w x y z) of `frames`, K ("body" | "site" | "geom",
        name) pairs; a name a model lacks gives NaN rows.  `touching` uint8/bool [n_envs]: touching_object of the geom
        `main_geom[slot]` names in model slot `slot` (None: 0); runs the full forward pass.  Tables are uploaded once
        per frame list / geom list."""
        t = self.torch
        d_frames = None
        if pose is not None:
            key = ("frames", tuple(frames))
            if key not in self._query_tables:
                tab = np.stack([lw.query_table(frames, TARGET_ALIAS.get(s.name, ()), MOVED_SITES.get(s.name))
                                for s, lw in zip(self.specs, self.lowered)])
                self._query_tables[key] = t.from_numpy(tab.view(np.uint8).reshape(-1).copy()).to(self.device)
            d_frames = self._query_tables[key]
        d_geom = None
        if touching is not None:
            if len(main_geom) != len(self.specs):
                raise ValueError(f"main_geom needs one entry per model slot ({len(self.specs)}), got {len(main_geom)}")
            key = ("geoms", tuple(main_geom))
            if key not in self._query_tables:
                g = [-1 if nm is None else lw.collider(nm) for nm, lw in zip(main_geom, self.lowered)]
                self._query_tables[key] = t.tensor(g, dtype=t.int32, device=self.device)
            d_geom = self._query_tables[key]
        _ck(lib().mw_query(self.h, self._p(mask), self._p(frame), self._p(d_frames), 0 if frames is None else len(frames),
                           self._p(pose), self._p(d_geom), self._p(touching), self._stream()))

    FAULTS = {1: "tolerance: lower bound > upper bound (the reference raises ValueError, reward_utils.py:124)",
              2: "tolerance: margin < 0 (the reference raises ValueError, reward_utils.py:134)",
              4: "hamacher_product: input outside [0, 1] (the reference raises ValueError, reward_utils.py:237)",
              8: "non-finite observation or reward",
              16: "stepped after its episode ended with autoreset disabled (reset it with reset_mask first; the reference's "
                  "SawyerXYZEnv.step raises ValueError past max_path_length)"}

    def faults(self):
        """Per-env MW_FAULT_* bits since the last call (cleared)."""
        out = np.zeros(self.n_envs, dtype=np.int32)
        self.torch.cuda.synchronize(self.device)
        _ck(lib().mw_get_faults(self.h, out.ctypes.data))
        return out

    def raise_on_faults(self):
        """Raises the reference's exception type for the first env that hit one of its error conditions."""
        f = self.faults()
        bad = np.nonzero(f)[0]
        if len(bad):
            e = int(bad[0])
            msgs = [m for b, m in self.FAULTS.items() if f[e] & b]
            raise ValueError(f"env {e}: " + "; ".join(msgs) + f" ({len(bad)} env(s) flagged)")

    def get_state(self):
        out = np.zeros(self.n_envs, dtype=ENVSTATE_DTYPE)
        self.torch.cuda.synchronize(self.device)
        _ck(lib().mw_get_state(self.h, out.ctypes.data))
        return out

    def set_state(self, st):
        st = np.ascontiguousarray(st, dtype=ENVSTATE_DTYPE)
        assert len(st) == self.n_envs
        self.torch.cuda.synchronize(self.device)
        _ck(lib().mw_set_state(self.h, st.ctypes.data))

    def debug_substeps(self, nstep, ctrl=(0.0, 0.0)):
        c = np.array(ctrl, dtype=np.float32)
        _ck(lib().mw_debug_substeps(self.h, int(nstep), c.ctypes.data, self._stream()))

    def debug_forward(self, ctrl=(0.0, 0.0)):
        """One forward pass per env without changing state; returns (contacts[n, MAXCON, 12], qacc[n, MAXDOF], meta[n, 4])."""
        nf = lib().mw_debug_dump_floats()
        buf = self.torch.zeros(self.n_envs, nf, device=self.device)
        c = np.array(ctrl, dtype=np.float32)
        _ck(lib().mw_debug_forward(self.h, c.ctypes.data, self._p(buf), self._stream()))
        a = buf.cpu().numpy()
        ncw = (nf - 17 - 4)
        return a[:, :ncw].reshape(self.n_envs, -1, 12), a[:, ncw:ncw + 17], a[:, ncw + 17:]

    PROFILE_KEYS = ["kin_mass", "collide", "gjk_epa", "constraints", "bias_smooth", "solver", "euler_glue", "obs_reward", "step",
                    "n_convex_pairs", "n_epa_expansions", "n_gjk_iters", "barrier_wait", "n_sep_tested", "n_sep_rejected"]

    def profile(self):
        """Per-phase warp-cycle counters summed over all env steps since the last call (mw_get_profile)."""
        out = np.zeros(len(self.PROFILE_KEYS), dtype=np.uint64)
        self.torch.cuda.synchronize(self.device)
        _ck(lib().mw_get_profile(self.h, out.ctypes.data))
        return dict(zip(self.PROFILE_KEYS, (int(x) for x in out)))

    def set_profiling(self, on=True):
        """Per-phase cycle counters are collected only while this is on (the timed kernel carries no profiling atomics)."""
        _ck(lib().mw_set_profiling(self.h, int(bool(on))))

    def env_profile(self):
        """[n_envs, 20] uint32: the first 13 PROFILE_KEYS for each env's last step, then [13] solver iterations, [14] ncon
        max, [15] nefc max, [16] launch slot, [17] convex pairs queued, [18] n_sep_tested, [19] n_sep_rejected."""
        out = np.zeros((self.n_envs, 20), dtype=np.uint32)
        self.torch.cuda.synchronize(self.device)
        _ck(lib().mw_get_env_profile(self.h, out.ctypes.data))
        return out

    def env_cost(self):
        out = np.zeros(self.n_envs, dtype=np.uint32)
        self.torch.cuda.synchronize(self.device)
        _ck(lib().mw_get_env_cost(self.h, out.ctypes.data))
        return out

    def rebalance(self):
        """Launch the costliest task types first (measured); see mw_rebalance."""
        _ck(lib().mw_rebalance(self.h))

    def counters(self):
        out = np.zeros(5, dtype=np.uint64)
        self.torch.cuda.synchronize(self.device)
        _ck(lib().mw_get_counters(self.h, out.ctypes.data))
        return dict(launches=int(out[0]), env_steps=int(out[1]), contacts_dropped=int(out[2]),
                    solver_iters=int(out[3]), forward_passes=int(out[4]))
