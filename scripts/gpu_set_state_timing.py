"""Device-timed state calls and a simulator-planning loop.

1. `set_state_torch(*get_state_torch())`, `get_state_torch()` and `observe_torch()` on all envs of MT50 x 4096 in steady
   state (episode phases staggered as in bench.py, 20 steps in), next to one `step_torch` of the same envs.
2. A CEM-style loop on one task: 64 root states x 64 candidate action sequences = 4096 envs.  Each iteration restores
   every env to its root (set_state_torch), reads the root observation (observe_torch) and rolls the candidates out for
   10 steps; the rate is env steps per second of the whole iteration.
Times come from CUDA events around `reps` back-to-back calls after a warm-up.  Prints one JSON line with the card name
and its power limit, and writes it to <out>/set_state_timing.json when an output directory is given.  Usage (on a GPU):
    python scripts/gpu_set_state_timing.py [reps] [out_dir]"""
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


def steady(name, use_one_hot):
    env = make_mt_envs(name, seed=42, num_envs=N, use_one_hot=use_one_hot)
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
    return env, acts


res = {"card": card(), "n_envs": N, "reps": REPS}
env, acts = steady("MT50", True)
qp, qv = env.get_state_torch()
k = [0]


def step():
    env.step_torch(acts[k[0] % 16]); k[0] += 1


res["mt50_ms"] = {"get_state_torch": timed(env.get_state_torch, REPS),
                  "set_state_torch": timed(lambda: env.set_state_torch(qp, qv), REPS),
                  "observe_torch": timed(env.observe_torch, REPS),
                  "step_torch": timed(step, max(10, REPS // 5))}
env.close()

# CEM-style planning: branch b (64 envs) restarts every iteration from root state b
task, H, B = "pick-place-v3", 10, 64
env, acts = steady(task, False)
qp, qv = env.get_state_torch()
root_q, root_v = qp[::B].repeat_interleave(B, 0).contiguous(), qv[::B].repeat_interleave(B, 0).contiguous()
plans = torch.rand(H, N, 4, device=env.device) * 2 - 1


def iteration():
    env.set_state_torch(root_q, root_v)
    env.observe_torch()
    for h in range(H):
        env.step_torch(plans[h])


it_ms = timed(iteration, max(5, REPS // 10), warm=2)
step_ms = timed(lambda: env.step_torch(plans[0]), max(10, REPS // 5))
res["cem"] = {"task": task, "branches": B, "candidates": N // B, "horizon": H, "iteration_ms": it_ms,
              "env_steps_per_s": N * H / (it_ms * 1e-3), "step_torch_ms_same_envs": step_ms}
assert not env.engine.faults().any()
env.close()
line = json.dumps(res)
print(line)
if OUT:
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "set_state_timing.json"), "w") as f:
        f.write(line + "\n")
