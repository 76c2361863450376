"""Benchmark definitions and task (goal) generation -- host side, run once at construction.

Mirrors the reference's registration layer: ``metaworld/env_dict.py`` (which env names make up
MT10/MT25/MT50 and the ML10/ML25/ML45 train/test splits; the order defines env ids / one-hot ids)
and ``metaworld/__init__.py:114-179`` (`_make_tasks`: the exact NumPy legacy-RNG protocol that turns a
seed into 50 goal vectors per env class).  `Task` keeps the reference's data format
(``metaworld/types.py:10-17``: env_name + pickled dict).
"""
from __future__ import annotations

import pickle
from dataclasses import dataclass

import numpy as np

from .tasks import TASKS

N_GOALS = 50  # metaworld/__init__.py:97

ALL_V3 = [
    "assembly-v3", "basketball-v3", "bin-picking-v3", "box-close-v3", "button-press-topdown-v3",
    "button-press-topdown-wall-v3", "button-press-v3", "button-press-wall-v3", "coffee-button-v3", "coffee-pull-v3",
    "coffee-push-v3", "dial-turn-v3", "disassemble-v3", "door-close-v3", "door-lock-v3", "door-open-v3",
    "door-unlock-v3", "hand-insert-v3", "drawer-close-v3", "drawer-open-v3", "faucet-open-v3", "faucet-close-v3",
    "hammer-v3", "handle-press-side-v3", "handle-press-v3", "handle-pull-side-v3", "handle-pull-v3", "lever-pull-v3",
    "pick-place-wall-v3", "pick-out-of-hole-v3", "pick-place-v3", "plate-slide-v3", "plate-slide-side-v3",
    "plate-slide-back-v3", "plate-slide-back-side-v3", "peg-insert-side-v3", "peg-unplug-side-v3", "soccer-v3",
    "stick-push-v3", "stick-pull-v3", "push-v3", "push-wall-v3", "push-back-v3", "reach-v3", "reach-wall-v3",
    "shelf-place-v3", "sweep-into-v3", "sweep-v3", "window-open-v3", "window-close-v3",
]
MT10 = ["reach-v3", "push-v3", "pick-place-v3", "door-open-v3", "drawer-open-v3", "drawer-close-v3",
        "button-press-topdown-v3", "peg-insert-side-v3", "window-open-v3", "window-close-v3"]
MT25 = MT10 + ["coffee-pull-v3", "pick-out-of-hole-v3", "disassemble-v3", "pick-place-wall-v3", "basketball-v3",
               "stick-pull-v3", "button-press-wall-v3", "faucet-open-v3", "door-lock-v3", "lever-pull-v3",
               "sweep-into-v3", "faucet-close-v3", "coffee-button-v3", "button-press-topdown-wall-v3", "dial-turn-v3"]
MT50 = list(ALL_V3)
ML10 = dict(train=["reach-v3", "push-v3", "pick-place-v3", "door-open-v3", "drawer-close-v3", "button-press-topdown-v3",
                   "peg-insert-side-v3", "window-open-v3", "sweep-v3", "basketball-v3"],
            test=["drawer-open-v3", "door-close-v3", "shelf-place-v3", "sweep-into-v3", "lever-pull-v3"])
ML25 = dict(train=list(MT25), test=["basketball-v3", "door-close-v3", "shelf-place-v3", "sweep-v3", "button-press-v3"])
ML45 = dict(train=["assembly-v3", "basketball-v3", "button-press-topdown-v3", "button-press-topdown-wall-v3",
                   "button-press-v3", "button-press-wall-v3", "coffee-button-v3", "coffee-pull-v3", "coffee-push-v3",
                   "dial-turn-v3", "disassemble-v3", "door-close-v3", "door-open-v3", "drawer-close-v3",
                   "drawer-open-v3", "faucet-open-v3", "faucet-close-v3", "hammer-v3", "handle-press-side-v3",
                   "handle-press-v3", "handle-pull-side-v3", "handle-pull-v3", "lever-pull-v3", "pick-place-wall-v3",
                   "pick-out-of-hole-v3", "push-back-v3", "pick-place-v3", "plate-slide-v3", "plate-slide-side-v3",
                   "plate-slide-back-v3", "plate-slide-back-side-v3", "peg-insert-side-v3", "peg-unplug-side-v3",
                   "soccer-v3", "stick-push-v3", "stick-pull-v3", "push-wall-v3", "push-v3", "reach-wall-v3",
                   "reach-v3", "shelf-place-v3", "sweep-into-v3", "sweep-v3", "window-open-v3", "window-close-v3"],
            test=["bin-picking-v3", "box-close-v3", "hand-insert-v3", "door-lock-v3", "door-unlock-v3"])


# reference env class of each task name (metaworld/env_dict.py:130-212: ALL_V3_ENVIRONMENTS); the checkpoint ids of the
# reference's CheckpointWrapper are f"{env_cls}_{env_id}" (metaworld/__init__.py:455), i.e. they embed repr(class)
REFERENCE_CLASS = {
    "assembly-v3": "metaworld.envs.sawyer_assembly_peg_v3.SawyerNutAssemblyEnvV3",
    "basketball-v3": "metaworld.envs.sawyer_basketball_v3.SawyerBasketballEnvV3",
    "bin-picking-v3": "metaworld.envs.sawyer_bin_picking_v3.SawyerBinPickingEnvV3",
    "box-close-v3": "metaworld.envs.sawyer_box_close_v3.SawyerBoxCloseEnvV3",
    "button-press-topdown-v3": "metaworld.envs.sawyer_button_press_topdown_v3.SawyerButtonPressTopdownEnvV3",
    "button-press-topdown-wall-v3": "metaworld.envs.sawyer_button_press_topdown_wall_v3.SawyerButtonPressTopdownWallEnvV3",
    "button-press-v3": "metaworld.envs.sawyer_button_press_v3.SawyerButtonPressEnvV3",
    "button-press-wall-v3": "metaworld.envs.sawyer_button_press_wall_v3.SawyerButtonPressWallEnvV3",
    "coffee-button-v3": "metaworld.envs.sawyer_coffee_button_v3.SawyerCoffeeButtonEnvV3",
    "coffee-pull-v3": "metaworld.envs.sawyer_coffee_pull_v3.SawyerCoffeePullEnvV3",
    "coffee-push-v3": "metaworld.envs.sawyer_coffee_push_v3.SawyerCoffeePushEnvV3",
    "dial-turn-v3": "metaworld.envs.sawyer_dial_turn_v3.SawyerDialTurnEnvV3",
    "disassemble-v3": "metaworld.envs.sawyer_disassemble_peg_v3.SawyerNutDisassembleEnvV3",
    "door-close-v3": "metaworld.envs.sawyer_door_close_v3.SawyerDoorCloseEnvV3",
    "door-lock-v3": "metaworld.envs.sawyer_door_lock_v3.SawyerDoorLockEnvV3",
    "door-open-v3": "metaworld.envs.sawyer_door_v3.SawyerDoorEnvV3",
    "door-unlock-v3": "metaworld.envs.sawyer_door_unlock_v3.SawyerDoorUnlockEnvV3",
    "hand-insert-v3": "metaworld.envs.sawyer_hand_insert_v3.SawyerHandInsertEnvV3",
    "drawer-close-v3": "metaworld.envs.sawyer_drawer_close_v3.SawyerDrawerCloseEnvV3",
    "drawer-open-v3": "metaworld.envs.sawyer_drawer_open_v3.SawyerDrawerOpenEnvV3",
    "faucet-open-v3": "metaworld.envs.sawyer_faucet_open_v3.SawyerFaucetOpenEnvV3",
    "faucet-close-v3": "metaworld.envs.sawyer_faucet_close_v3.SawyerFaucetCloseEnvV3",
    "hammer-v3": "metaworld.envs.sawyer_hammer_v3.SawyerHammerEnvV3",
    "handle-press-side-v3": "metaworld.envs.sawyer_handle_press_side_v3.SawyerHandlePressSideEnvV3",
    "handle-press-v3": "metaworld.envs.sawyer_handle_press_v3.SawyerHandlePressEnvV3",
    "handle-pull-side-v3": "metaworld.envs.sawyer_handle_pull_side_v3.SawyerHandlePullSideEnvV3",
    "handle-pull-v3": "metaworld.envs.sawyer_handle_pull_v3.SawyerHandlePullEnvV3",
    "lever-pull-v3": "metaworld.envs.sawyer_lever_pull_v3.SawyerLeverPullEnvV3",
    "pick-place-wall-v3": "metaworld.envs.sawyer_pick_place_wall_v3.SawyerPickPlaceWallEnvV3",
    "pick-out-of-hole-v3": "metaworld.envs.sawyer_pick_out_of_hole_v3.SawyerPickOutOfHoleEnvV3",
    "pick-place-v3": "metaworld.envs.sawyer_pick_place_v3.SawyerPickPlaceEnvV3",
    "plate-slide-v3": "metaworld.envs.sawyer_plate_slide_v3.SawyerPlateSlideEnvV3",
    "plate-slide-side-v3": "metaworld.envs.sawyer_plate_slide_side_v3.SawyerPlateSlideSideEnvV3",
    "plate-slide-back-v3": "metaworld.envs.sawyer_plate_slide_back_v3.SawyerPlateSlideBackEnvV3",
    "plate-slide-back-side-v3": "metaworld.envs.sawyer_plate_slide_back_side_v3.SawyerPlateSlideBackSideEnvV3",
    "peg-insert-side-v3": "metaworld.envs.sawyer_peg_insertion_side_v3.SawyerPegInsertionSideEnvV3",
    "peg-unplug-side-v3": "metaworld.envs.sawyer_peg_unplug_side_v3.SawyerPegUnplugSideEnvV3",
    "soccer-v3": "metaworld.envs.sawyer_soccer_v3.SawyerSoccerEnvV3",
    "stick-push-v3": "metaworld.envs.sawyer_stick_push_v3.SawyerStickPushEnvV3",
    "stick-pull-v3": "metaworld.envs.sawyer_stick_pull_v3.SawyerStickPullEnvV3",
    "push-v3": "metaworld.envs.sawyer_push_v3.SawyerPushEnvV3",
    "push-wall-v3": "metaworld.envs.sawyer_push_wall_v3.SawyerPushWallEnvV3",
    "push-back-v3": "metaworld.envs.sawyer_push_back_v3.SawyerPushBackEnvV3",
    "reach-v3": "metaworld.envs.sawyer_reach_v3.SawyerReachEnvV3",
    "reach-wall-v3": "metaworld.envs.sawyer_reach_wall_v3.SawyerReachWallEnvV3",
    "shelf-place-v3": "metaworld.envs.sawyer_shelf_place_v3.SawyerShelfPlaceEnvV3",
    "sweep-into-v3": "metaworld.envs.sawyer_sweep_into_goal_v3.SawyerSweepIntoGoalEnvV3",
    "sweep-v3": "metaworld.envs.sawyer_sweep_v3.SawyerSweepEnvV3",
    "window-open-v3": "metaworld.envs.sawyer_window_open_v3.SawyerWindowOpenEnvV3",
    "window-close-v3": "metaworld.envs.sawyer_window_close_v3.SawyerWindowCloseEnvV3",
}


def reference_env_id(task_name, env_id):
    """The string the reference passes to CheckpointWrapper(env, f"{env_cls}_{env_id}") (metaworld/__init__.py:455)."""
    return f"<class '{REFERENCE_CLASS[task_name]}'>_{env_id}"


class _RefModule:
    """Pickles as ``importlib.import_module(name)``."""

    def __init__(self, name):
        self.name = name

    def __reduce__(self):
        import importlib
        return (importlib.import_module, (self.name,))


class _RefClass:
    """Pickles as ``getattr(importlib.import_module(module), name)``: a task made here unpickles, inside the reference
    package, to the reference's env class, which is what ``SawyerXYZEnv.set_task`` asserts on (sawyer_xyz_env.py:306) --
    so checkpoints and Task lists written by this package load in the reference unchanged."""

    def __init__(self, dotted):
        self.module, self.name = dotted.rsplit(".", 1)

    def __reduce__(self):
        return (getattr, (_RefModule(self.module), self.name))


class _MissingModule:
    def __init__(self, name):
        self._name = name

    def __getattr__(self, k):
        return f"{self._name}.{k}"


def _import_or_placeholder(name):
    import importlib
    try:
        return importlib.import_module(name)
    except Exception:
        return _MissingModule(name)


@dataclass
class Task:
    """Same shape as the reference's ``metaworld.types.Task``: ``data`` is a pickled dict with
    ``rand_vec``, ``env_cls`` (here: the env name string) and ``partially_observable``."""
    env_name: str
    data: bytes

    def unpack(self):
        """The pickled dict.  Tasks made by the reference pickle ``env_cls`` as a class object
        (metaworld/__init__.py:171); where that package is not importable the class is read back as its dotted name."""
        import io

        cached = self.__dict__.get("_unpacked")
        if cached is not None:
            return cached

        class _U(pickle.Unpickler):
            def find_class(self, module, name):
                if (module, name) == ("importlib", "import_module"):
                    return _import_or_placeholder
                try:
                    return super().find_class(module, name)
                except Exception:
                    return f"{module}.{name}"

        self.__dict__["_unpacked"] = d = _U(io.BytesIO(self.data)).load()     # cached: the hot autoreset path asks per episode
        return d


def draw_rand_vec(spec, rs: np.random.RandomState):
    """One ``reset_model`` worth of ``_get_state_rand_vec`` calls with ``_freeze_rand_vec=False``
    (sawyer_xyz_env.py:709-719 + the task's rejection loop, e.g. sawyer_reach_v3.py:125-129)."""
    lo, hi = spec.rand_low, spec.rand_high
    v = rs.uniform(lo, hi, size=lo.size).astype(np.float64)
    if spec.reject is not None:
        (a0, a1), other, thr = spec.reject

        def ref(v):   # either another slice of the vector or a fixed point (sweep-into: the constant goal)
            return v[other[0]:other[1]] if isinstance(other[0], int) else np.asarray(other)

        while np.linalg.norm(v[a0:a1] - ref(v)) < thr:
            v = rs.uniform(lo, hi, size=lo.size).astype(np.float64)
    return v


def make_tasks(env_names, partially_observable: bool, seed=None, n_goals=N_GOALS):
    """``_make_tasks`` (metaworld/__init__.py:114-179): per env class, ``n_goals`` resets with an unfrozen
    rand_vec; every reset runs ``reset_model`` twice (sawyer_xyz_env.py:677-678) so two draws happen per goal
    and the second one is kept."""
    rs = np.random.RandomState(seed) if seed is not None else np.random.RandomState()
    tasks = []
    for name in env_names:
        spec = TASKS[name]
        vecs = []
        for _ in range(n_goals):
            draw_rand_vec(spec, rs)           # pass 1 (discarded)
            vecs.append(draw_rand_vec(spec, rs))  # pass 2
        if len(np.unique(np.array(vecs), axis=0)) != n_goals:
            raise AssertionError(f"Only generated {len(np.unique(np.array(vecs), axis=0))} unique goals, not {n_goals}")
        for v in vecs:
            tasks.append(make_task(name, v, partially_observable))
    return tasks


def make_task(name, rand_vec, partially_observable: bool):
    """The reference's ``Task`` of env class `name` with goal vector `rand_vec` (metaworld/__init__.py:171)."""
    return Task(name, pickle.dumps(dict(rand_vec=rand_vec, env_cls=_RefClass(REFERENCE_CLASS[name]), partially_observable=partially_observable)))


class EnvClass:
    """Stands where the reference keeps an env CLASS (``benchmark.train_classes[name]``, metaworld/__init__.py:184-196):
    calling it builds the bare single env over the engine (metaworld_b200.single_env.SawyerXYZEnvB200)."""

    def __init__(self, env_name):
        self.env_name = env_name
        self.__name__ = REFERENCE_CLASS[env_name].rsplit(".", 1)[1]

    def __call__(self, *a, **k):
        from .single_env import SawyerXYZEnvB200
        return SawyerXYZEnvB200(self.env_name, *a, **k)

    def __repr__(self):
        return f"<class '{REFERENCE_CLASS[self.env_name]}'>"


def _classes(names):
    from collections import OrderedDict
    return OrderedDict((n, EnvClass(n)) for n in names)


class Benchmark:
    """``metaworld.Benchmark`` surface: train_classes / test_classes (OrderedDict name -> env class, iterates as the
    names) and train_tasks / test_tasks."""

    def __init__(self, train, test, partially_observable, seed, test_seed=None, n_goals=N_GOALS):
        self.train_classes = _classes(train)
        self.test_classes = _classes(test)
        self.train_tasks = make_tasks(train, partially_observable, seed, n_goals)
        self.test_tasks = make_tasks(test, partially_observable, seed if test_seed is None else test_seed, n_goals) if test else []


def MT1(env_name, seed=None, n_goals=N_GOALS):
    b = Benchmark([env_name], [], False, seed, n_goals=n_goals)
    b.test_classes = _classes([env_name])
    return b


def ML1(env_name, seed=None, n_goals=N_GOALS):
    return Benchmark([env_name], [env_name], True, seed, test_seed=(seed + 1 if seed is not None else None), n_goals=n_goals)


def make_benchmark(name, seed=None, n_goals=N_GOALS):
    """``num_goals`` of the reference's entry points rebinds its module-global _N_GOALS (metaworld/__init__.py:620-623)."""
    if name in TASKS or name in ALL_V3:
        return MT1(name, seed, n_goals)
    table = dict(MT10=(MT10, [], False), MT25=(MT25, [], False), MT50=(MT50, [], False),
                 ML10=(ML10["train"], ML10["test"], True), ML25=(ML25["train"], ML25["test"], True),
                 ML45=(ML45["train"], ML45["test"], True))
    if name not in table:
        raise ValueError(f"unknown benchmark {name!r}")
    tr, te, po = table[name]
    return Benchmark(tr, te, po, seed, n_goals=n_goals)
