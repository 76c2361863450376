"""Evaluation loops over a `MetaWorldVecEnv` -- same signatures, return values and bookkeeping as the reference's
``metaworld/evaluation.py:48-169`` (`evaluation`, `metalearning_evaluation`, the `Agent` / `MetaLearningAgent` protocols and
`Timestep`), with the per-env Python loops replaced by array operations so that 4096-env evaluations stay cheap on the
host.  Works with any object that follows the vector-env protocol used there (`reset`, `step`, `call`, `get_attr`,
`num_envs`), which is what the CPU test drives it with.
"""
from __future__ import annotations

from typing import NamedTuple, Protocol

import numpy as np


class Agent(Protocol):
    def eval_action(self, observations: np.ndarray) -> np.ndarray: ...
    def reset(self, env_mask: np.ndarray) -> None: ...


class MetaLearningAgent(Agent, Protocol):
    def init(self) -> None: ...
    def adapt_action(self, observations: np.ndarray) -> tuple[np.ndarray, dict[str, np.ndarray]]: ...
    def step(self, timestep: "Timestep") -> None: ...
    def adapt(self) -> None: ...


class Timestep(NamedTuple):
    observation: np.ndarray
    action: np.ndarray
    reward: np.ndarray
    terminated: np.ndarray
    truncated: np.ndarray
    aux_policy_outputs: dict


def _get_task_names(envs) -> list[str]:
    """One task name per sub-env (the reference maps env classes back to names, evaluation.py:38-45)."""
    return [str(n) for n in envs.get_attr("task_name")]


def evaluation(agent: Agent, eval_envs, num_episodes: int = 50):
    """evaluation.py:48-105: run until every task has `num_episodes` finished episodes; successes are counted on the first
    `num_episodes` episodes of each task (in order of completion, env index breaking ties within a step), returns are the
    first `num_episodes` episodic returns per task.  Like the reference, it reads `final_info`, so `eval_envs` must use the
    default SAME_STEP autoreset."""
    terminate_on_success = bool(np.all(eval_envs.get_attr("terminate_on_success")))
    eval_envs.call("toggle_terminate_on_success", True)
    obs, _ = eval_envs.reset()
    agent.reset(np.ones(eval_envs.num_envs, dtype=np.bool_))
    task_names = _get_task_names(eval_envs)
    uniq = list(dict.fromkeys(task_names))
    tid = np.array([uniq.index(n) for n in task_names])
    successes = np.zeros(len(uniq), dtype=np.int64)
    counts = np.zeros(len(uniq), dtype=np.int64)
    returns: list[list[float]] = [[] for _ in uniq]
    while counts.min() < num_episodes:
        actions = agent.eval_action(obs)
        obs, _, terminations, truncations, infos = eval_envs.step(actions)
        dones = np.logical_or(terminations, truncations)
        agent.reset(dones)
        if dones.any():
            idx = np.nonzero(dones)[0]                                   # ascending env index = the reference's loop order
            ep_r = np.asarray(infos["final_info"]["episode"]["r"], dtype=np.float64)[idx]
            succ = np.asarray(infos["final_info"]["success"])[idx].astype(np.int64)
            t = tid[idx]
            for k in np.unique(t):
                sel = t == k
                r_k, s_k = ep_r[sel], succ[sel]
                room = max(0, num_episodes - counts[k])                 # only the first num_episodes episodes count for success
                successes[k] += int(s_k[:room].sum())
                counts[k] += len(r_k)
                returns[k].extend(float(x) for x in r_k)
    episodic_returns = {n: returns[k][:num_episodes] for k, n in enumerate(uniq)}
    success_rate_per_task = {n: successes[k] / num_episodes for k, n in enumerate(uniq)}
    mean_success_rate = float(np.mean(list(success_rate_per_task.values())))
    mean_returns = float(np.mean(list(episodic_returns.values())))
    eval_envs.call("toggle_terminate_on_success", terminate_on_success)
    return mean_success_rate, mean_returns, success_rate_per_task, episodic_returns


def metalearning_evaluation(agent: MetaLearningAgent, eval_envs, num_evals: int = 10, adaptation_steps: int = 1,
                            adaptation_episodes: int = 10, evaluation_episodes: int = 3):
    """evaluation.py:108-169: per evaluation round sample new tasks, let the agent adapt for `adaptation_steps` x
    `adaptation_episodes` episodes per env, then run `evaluation`."""
    eval_envs.call("toggle_sample_tasks_on_reset", False)
    eval_envs.call("toggle_terminate_on_success", False)
    task_names = _get_task_names(eval_envs)
    uniq = list(dict.fromkeys(task_names))
    total_sr = total_ret = 0.0
    sr_per_task = np.zeros((num_evals, len(uniq)))
    for i in range(num_evals):
        eval_envs.call("sample_tasks")
        agent.init()
        for _ in range(adaptation_steps):
            obs, _ = eval_envs.reset()
            episodes_elapsed = np.zeros((eval_envs.num_envs,), dtype=np.uint16)
            while not (episodes_elapsed >= adaptation_episodes).all():
                actions, aux = agent.adapt_action(obs)
                next_obs, rewards, terminations, truncations, _ = eval_envs.step(actions)
                agent.step(Timestep(obs, actions, rewards, terminations, truncations, aux))
                episodes_elapsed += np.logical_or(terminations, truncations)
                obs = next_obs
            agent.adapt()
        sr, ret, per_task, _ = evaluation(agent, eval_envs, evaluation_episodes)
        total_sr += sr
        total_ret += ret
        sr_per_task[i] = np.array([per_task[n] for n in uniq])
    rates = sr_per_task.mean(axis=0)
    return total_sr / num_evals, total_ret / num_evals, {n: float(rates[k]) for k, n in enumerate(uniq)}
