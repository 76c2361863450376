"""Device-timed scripted expert policies (`expert_actions_torch`, kernel k_expert).

1. `expert_actions_torch()` on all envs of MT50 x 4096 in steady state (episode phases staggered as in bench.py, 20 steps
   in), next to one `step_torch` of the same envs.
2. Demonstration collection: `step_torch(expert_actions_torch())` closed loop against `step_torch` with precomputed
   actions, in env steps per second.
Times come from CUDA events around `reps` back-to-back calls after a warm-up.  Prints one JSON line with the card name
and its power limit, and writes it to <out>/expert_timing.json when an output directory is given.  Usage (on a GPU):
    python scripts/gpu_expert_timing.py [reps] [out_dir]"""
import json, os, sys

import numpy as np
import torch

from gpu_timing_common import card, steady_env, timed

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 100
OUT = sys.argv[2] if len(sys.argv) > 2 else None
N = 4096


env = steady_env("MT50", N, use_one_hot=True)
rng = np.random.default_rng(1)
acts = [torch.from_numpy(rng.uniform(-1, 1, size=(N, 4)).astype(np.float32)).cuda() for _ in range(16)]
for i in range(20):
    env.step_torch(acts[i % 16])

res = {"card": card(), "n_envs": N, "reps": REPS}
res["expert_actions_torch_ms"] = timed(lambda: env.expert_actions_torch(), REPS)
k = [0]


def step_fixed():
    env.step_torch(acts[k[0] % 16]); k[0] += 1


res["step_torch_ms"] = timed(step_fixed, REPS)
res["collect_ms_per_step"] = timed(lambda: env.step_torch(env.expert_actions_torch()), REPS)
res["collect_env_steps_per_s"] = N / (res["collect_ms_per_step"] * 1e-3)
res["fixed_actions_env_steps_per_s"] = N / (res["step_torch_ms"] * 1e-3)
print(json.dumps(res))
if OUT:
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "expert_timing.json"), "w") as f:
        json.dump(res, f, indent=1)
env.close()
