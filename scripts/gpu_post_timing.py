"""Time of the numpy `step` and of `step_torch` with the optional per-env wrappers on (recurrent observation, gymnasium
reward normalisation, observation normalisation), which bench.py's workload leaves off: MT50 @ 4096 envs, episode phases
staggered as in bench.py so that every step finishes a few episodes.  Prints one JSON line with the card name, its power
limit and max SM clock.  Usage (on a GPU):
    python scripts/gpu_post_timing.py [steps]"""
import json, sys, time

import numpy as np
import torch

from gpu_timing_common import card, steady_env

STEPS = int(sys.argv[1]) if len(sys.argv) > 1 else 200
N = 4096
env = steady_env("MT50", N, use_one_hot=True, recurrent_info_in_obs=True, reward_normalization_method="gymnasium",
                 normalize_observations=True)
rng = np.random.default_rng(1)
acts = [rng.uniform(-1, 1, size=(N, 4)).astype(np.float32) for _ in range(16)]
for i in range(50):
    env.step(acts[i % 16])
t0 = time.perf_counter()
for i in range(STEPS):
    env.step(acts[i % 16])               # returns host arrays: ends in a device synchronise
step_ms = (time.perf_counter() - t0) / STEPS * 1e3
d_acts = [torch.from_numpy(a).to(env.device) for a in acts]
for i in range(50):
    env.step_torch(d_acts[i % 16])
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
t0 = time.perf_counter()
e0.record()
for i in range(STEPS):
    env.step_torch(d_acts[i % 16])
e1.record()
torch.cuda.synchronize()
wall_ms = (time.perf_counter() - t0) / STEPS * 1e3
print(json.dumps(dict(card=card(), envs=N, steps=STEPS, step_ms=round(step_ms, 3),
                      step_torch_device_ms=round(e0.elapsed_time(e1) / STEPS, 3), step_torch_wall_ms=round(wall_ms, 3))))
env.close()
