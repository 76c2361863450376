"""Device-timed `step_torch` at MT50 x 4096 envs in steady state under each autoreset mode (SAME_STEP, NEXT_STEP, and
DISABLED with `reset_torch(reset_mask=terminated | truncated)` after every step, both timed).  Episode phases are
staggered as in bench.py so that every step ends a few episodes.  The modes run alternately, `rounds` times, in one
process.  Prints one JSON line with the card name and its power limit.  Usage (on a GPU):
    python scripts/gpu_autoreset_timing.py [steps] [rounds]"""
import json, os, subprocess, sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from metaworld_b200.vector_env import make_mt_envs  # noqa: E402

STEPS = int(sys.argv[1]) if len(sys.argv) > 1 else 200
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 3
N = 4096
MODES = ("SameStep", "NextStep", "Disabled")
rng = np.random.default_rng(1)
d_acts = [torch.from_numpy(rng.uniform(-1, 1, size=(N, 4)).astype(np.float32)).cuda() for _ in range(16)]


def make(mode):
    env = make_mt_envs("MT50", seed=42, num_envs=N, use_one_hot=True, autoreset_mode=mode)
    env.reset_torch()
    p = (np.arange(N) * 500 // N)[np.random.default_rng(0).permutation(N)]          # bench.stagger
    st = env.engine.get_state()
    st["path_len"] = p.astype(np.float32)
    env.engine.set_state(st)
    env._ep_len[:] = p
    return env


def run(env, mode, steps):
    for i in range(steps):
        _, _, te, tr, _ = env.step_torch(d_acts[i % 16])
        if mode == "Disabled":
            env.reset_torch((te | tr).bool())


envs = {m: make(m) for m in MODES}
for m in MODES:
    run(envs[m], m, 100)                 # warm-up: launch order and episode phases reach steady state
torch.cuda.synchronize()
ms = {m: [] for m in MODES}
for r in range(ROUNDS):
    for m in MODES:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run(envs[m], m, STEPS)
        e1.record()
        torch.cuda.synchronize()
        ms[m].append(round(e0.elapsed_time(e1) / STEPS, 4))
try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30).stdout.strip()
except Exception:  # noqa: BLE001 -- reported as unknown
    power = "unknown"
print(json.dumps(dict(device=torch.cuda.get_device_name(), power_limit=power, envs=N, steps=STEPS, rounds=ROUNDS,
                      step_torch_device_ms=ms, median_ms={m: float(np.median(v)) for m, v in ms.items()})))
for e in envs.values():
    e.close()
