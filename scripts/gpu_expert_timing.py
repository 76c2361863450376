"""Device-timed scripted expert policies (`expert_actions_torch`, kernel k_expert).

1. `expert_actions_torch()` on all envs of MT50 x 4096 in steady state (episode phases staggered as in bench.py, 20 steps
   in), next to one `step_torch` of the same envs.
2. Demonstration collection: `step_torch(expert_actions_torch())` closed loop against `step_torch` with precomputed
   actions, in env steps per second.
Times come from CUDA events around `reps` back-to-back calls after a warm-up.  Prints one JSON line with the card name
and its power limit, and writes it to <out>/expert_timing.json when an output directory is given.  Usage (on a GPU):
    python scripts/gpu_expert_timing.py [reps] [out_dir]"""
import json, os, subprocess, sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from metaworld_b200.vector_env import make_mt_envs  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 100
OUT = sys.argv[2] if len(sys.argv) > 2 else None
N = 4096


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q[0] if q else None}


def timed(fn, reps, warm=5):
    for _ in range(warm):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


env = make_mt_envs("MT50", seed=42, num_envs=N, use_one_hot=True)
env.reset()
p = (np.arange(N) * 500 // N)[np.random.default_rng(0).permutation(N)]          # bench.stagger
st = env.engine.get_state()
st["path_len"] = p.astype(np.float32)
env.engine.set_state(st)
env._ep_len[:] = p
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
