"""metaworld_b200: H100-native batched Meta-World step engine (see DESIGN.md).

Public surface mirrors the reference package (``metaworld/__init__.py``): ``make_mt_envs`` / ``make_ml_envs``, the
benchmark classes, ``evaluation`` and -- when gymnasium is installed -- every id the reference registers
(``MT1 | MT10 | MT25 | MT50 | ML1-* | ML10-* | ML25-* | ML45-* | goal_hidden | goal_observable | custom-mt-envs |
custom-ml-envs``, metaworld/__init__.py:607-820).  The ids live in the namespace ``Meta-World-B200/`` so both packages can
coexist; ``register_mw_envs(stock_ids=True)`` (or METAWORLD_B200_STOCK_IDS=1 in the environment) additionally claims the
reference's own ``Meta-World/...`` ids, which is the drop-in switch: user code calling ``gym.make_vec("Meta-World/MT50",
...)`` then runs on the engine unchanged."""
from __future__ import annotations

import os

__version__ = "0.2.0"

from .benchmarks import ALL_V3, ML1, ML10, ML25, ML45, MT1, MT10, MT25, MT50, Benchmark, Task, make_benchmark  # noqa: F401
from . import evaluation  # noqa: F401  (evaluation / metalearning_evaluation, metaworld/evaluation.py)
from . import policies  # noqa: F401  (ENV_POLICY_MAP, the scripted expert policies, metaworld/policies/__init__.py)


def make_mt_envs(*a, **k):
    from .vector_env import make_mt_envs as f
    return f(*a, **k)


def make_ml_envs(*a, **k):
    from .vector_env import make_ml_envs as f
    return f(*a, **k)


def entry_points():
    """id suffix -> (entry_point, vector_entry_point), argument names as in the reference's lambdas."""
    from . import vector_env as V
    from . import single_env as S

    def mt(name):
        def vec(seed=None, use_one_hot=False, num_envs=None, vector_strategy="sync", autoreset_mode=None, **kw):
            return V.make_mt_envs(name, seed=seed, use_one_hot=use_one_hot, num_envs=num_envs, autoreset_mode=autoreset_mode, **kw)
        return vec

    def ml(name, split):
        def vec(seed=None, meta_batch_size=20, total_tasks_per_cls=None, num_envs=None, vector_strategy="sync", autoreset_mode=None, **kw):
            # make_ml_envs_train / _test partials (metaworld/__init__.py:596-604)
            kw.setdefault("terminate_on_success", split == "test")
            return V.make_ml_envs(kw.pop("env_name", name), seed=seed, meta_batch_size=meta_batch_size, total_tasks_per_cls=total_tasks_per_cls,
                                  split=split, num_envs=num_envs, autoreset_mode=autoreset_mode, **kw)
        return vec

    def mt1_single(env_name, use_one_hot=False, seed=None, num_envs=None, vector_strategy="sync", autoreset_mode=None, **kw):
        return V.make_mt_envs(env_name, seed=seed, use_one_hot=use_one_hot, single=True, **kw)      # gym.make -> ONE wrapped env

    def mt1_vec(env_name, use_one_hot=False, seed=None, num_envs=None, vector_strategy="sync", autoreset_mode=None, **kw):
        return V.make_mt_envs(env_name, seed=seed, use_one_hot=use_one_hot, num_envs=num_envs, autoreset_mode=autoreset_mode, **kw)

    table = {"MT1": (mt1_single, mt1_vec)}
    for n in ("MT10", "MT25", "MT50"):
        table[n] = (None, mt(n))
    for n in ("ML1", "ML10", "ML25", "ML45"):
        for split in ("train", "test"):
            table[f"{n}-{split}"] = (None, ml(n, split))
    table["goal_hidden"] = (lambda env_name, seed=None, **kw: S.make_goal_env(env_name, seed, observable=False, **kw), None)
    table["goal_observable"] = (lambda env_name, seed=None, **kw: S.make_goal_env(env_name, seed, observable=True, **kw), None)
    table["custom-mt-envs"] = (None, lambda envs_list, seed=None, use_one_hot=False, num_envs=None, vector_strategy="sync", autoreset_mode=None, **kw:
                               V.make_custom_mt_envs(envs_list, seed=seed, use_one_hot=use_one_hot, num_envs=num_envs, autoreset_mode=autoreset_mode, **kw))
    table["custom-ml-envs"] = (None, lambda train_envs, test_envs, seed=None, meta_batch_size=20, total_tasks_per_cls=None, num_envs=None,
                               vector_strategy="sync", autoreset_mode=None, **kw:
                               V.make_custom_ml_envs(train_envs, test_envs, seed=seed, meta_batch_size=meta_batch_size,
                                                     total_tasks_per_cls=total_tasks_per_cls, num_envs=num_envs, autoreset_mode=autoreset_mode,
                                                     **kw))
    return table


def register_mw_envs(stock_ids=None):
    """gymnasium registration (metaworld/__init__.py:607-820) when gymnasium is available.  Returns the ids registered."""
    from . import _gym
    if not _gym.HAVE_GYMNASIUM:
        return []
    from gymnasium.envs.registration import register

    if stock_ids is None:
        stock_ids = os.environ.get("METAWORLD_B200_STOCK_IDS", "0") == "1"
    done = []
    for ns in (["Meta-World-B200"] + (["Meta-World"] if stock_ids else [])):
        for suffix, (single, vec) in entry_points().items():
            kw = {}
            if single is not None:
                kw["entry_point"] = single
            if vec is not None:
                kw["vector_entry_point"] = vec
            register(id=f"{ns}/{suffix}", kwargs={}, **kw)
            done.append(f"{ns}/{suffix}")
    return done


try:
    register_mw_envs()
except Exception:  # registration is best effort
    pass
