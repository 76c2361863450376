"""Device-timed open-loop rollouts (k_rollout) against the fork-and-step loop they replace, on the same env steps.

1. MPPI shape: pick-place-v3, 64 envs, K = 64 candidates, H = 30 steps with `rollout_torch`, against the existing loop on
   4096 envs (64 sources x 64 branches): a `load_states_torch` fork, then 30 `step_torch` calls.
2. Fusion alone: MT50 x 4096 in steady state (episode phases staggered as in bench.py, 20 steps in), K = 1, H = 30, against
   `load_states_torch` of the state saved before followed by 30 `step_torch` calls of the same actions.
3. Kernel only: CUDA events around the engine call (`Engine.rollout` into caller-owned buffers) of both shapes.
Times come from CUDA events around back-to-back calls after a warm-up of every shape; the compared variants alternate
`rounds` times in one session and every time is reported.  Prints one JSON line with the card name, its power limit and max
SM clock, and writes it to <out>/rollout_timing.json when an output directory is given.  Usage (on a GPU):
    python scripts/gpu_rollout_timing.py [reps] [out_dir]"""
import json, os, sys

import numpy as np
import torch

from gpu_timing_common import card, steady_env, timed

REPS = max(10, int(sys.argv[1]) if len(sys.argv) > 1 else 20)
OUT = sys.argv[2] if len(sys.argv) > 2 else None
ROUNDS = 3
H = 30


def steady(name, n, use_one_hot=False):
    env = steady_env(name, n, use_one_hot=use_one_hot)
    rng = np.random.default_rng(1)
    for _ in range(20):
        env.step_torch(torch.from_numpy(rng.uniform(-1, 1, size=(n, 4)).astype(np.float32)).cuda())
    return env


def engine_call(env, actions):
    """The bare engine call of `rollout_torch` with preallocated outputs (no observations)."""
    K, n = actions.shape[0], env.num_envs
    out = (torch.empty(K, H, n, device="cuda"), torch.empty(K, H, n, 7, device="cuda"),
           torch.empty(K, H, n, dtype=torch.uint8, device="cuda"), None, torch.empty(K, n, 2, dtype=torch.int32, device="cuda"),
           torch.empty(K * n, 128, 4, device="cuda"))
    return lambda: env.engine.rollout(actions, *out)


def alternate(variants, reps):
    """{name: [ms per call, one per round]} with the variants timed in turn, `ROUNDS` times."""
    res = {k: [] for k in variants}
    for _ in range(ROUNDS):
        for k, fn in variants.items():
            res[k].append(timed(fn, reps, warm=2))
    return res


res = {"card": card(), "horizon": H, "reps": REPS, "rounds": ROUNDS}

# 1. MPPI shape
task, B, n = "pick-place-v3", 64, 64
small, big = steady(task, n), steady(task, n * B)
acts = torch.rand(B, H, n, 4, device="cuda") * 2 - 1                 # candidate k of env s = branch k of source s
plans = acts.permute(1, 2, 0, 3).reshape(H, n * B, 4).contiguous()   # the same actions on the 4096-env table
st = big.save_states()
src = (torch.arange(n * B, device="cuda") // B) * B


def fork_and_step():
    big.load_states_torch(st, src=src)
    for h in range(H):
        big.step_torch(plans[h])


t = alternate({"rollout_torch": lambda: small.rollout_torch(acts), "fork_and_step": fork_and_step,
               "engine_rollout": engine_call(small, acts)}, REPS)
steps = n * B * H
res["mppi"] = {"task": task, "envs": n, "candidates": B, "fork_envs": n * B, "env_steps_per_call": steps, "ms": t,
               "env_steps_per_s": {k: steps / (min(v) * 1e-3) for k, v in t.items()},
               "rollout_over_fork_and_step": min(t["rollout_torch"]) / min(t["fork_and_step"])}
assert not small.engine.faults().any() and not big.engine.faults().any()
small.close(); big.close()

# 2. fusion alone
n = 4096
env = steady("MT50", n, use_one_hot=True)
acts = torch.rand(1, H, n, 4, device="cuda") * 2 - 1
st = env.save_states()


def load_and_step():
    env.load_states_torch(st)
    for h in range(H):
        env.step_torch(acts[0, h])


t = alternate({"rollout_torch": lambda: env.rollout_torch(acts), "load_and_step": load_and_step,
               "engine_rollout": engine_call(env, acts)}, REPS)
steps = n * H
res["mt50_fusion"] = {"envs": n, "candidates": 1, "env_steps_per_call": steps, "ms": t,
                      "ms_per_env_step_slice": {k: min(v) / H for k, v in t.items()},
                      "rollout_over_load_and_step": min(t["rollout_torch"]) / min(t["load_and_step"])}
assert not env.engine.faults().any()
env.close()

line = json.dumps(res)
print(line)
if OUT:
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "rollout_timing.json"), "w") as f:
        f.write(line + "\n")
