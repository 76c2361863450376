"""Device-timed `step_torch` at MT50 x 4096 envs in steady state under each autoreset mode (SAME_STEP, NEXT_STEP, and
DISABLED with `reset_torch(reset_mask=terminated | truncated)` after every step, both timed).  Episode phases are
staggered as in bench.py so that every step ends a few episodes.  The modes run alternately, `rounds` times, in one
process.  Prints one JSON line with the card name, its power limit and max SM clock.  Usage (on a GPU):
    python scripts/gpu_autoreset_timing.py [steps] [rounds]"""
import json, sys

import numpy as np
import torch

from gpu_timing_common import card, steady_env

STEPS = int(sys.argv[1]) if len(sys.argv) > 1 else 200
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 3
N = 4096
MODES = ("SameStep", "NextStep", "Disabled")
rng = np.random.default_rng(1)
d_acts = [torch.from_numpy(rng.uniform(-1, 1, size=(N, 4)).astype(np.float32)).cuda() for _ in range(16)]


def run(env, mode, steps):
    for i in range(steps):
        _, _, te, tr, _ = env.step_torch(d_acts[i % 16])
        if mode == "Disabled":
            env.reset_torch((te | tr).bool())


envs = {m: steady_env("MT50", N, use_one_hot=True, autoreset_mode=m) for m in MODES}
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
print(json.dumps(dict(card=card(), envs=N, steps=STEPS, rounds=ROUNDS,
                      step_torch_device_ms=ms, median_ms={m: float(np.median(v)) for m, v in ms.items()})))
for e in envs.values():
    e.close()
