"""Device-timed episodes at new goals (k_goal_rows + k_reset_rows through `reset_goals_torch`).

1. MT50 x 4096 in steady state (episode phases staggered as in bench.py, 20 steps in): `reset_goals_torch` of every env
   and of 8 random envs (about N / 500, the number of episodes that end in one steady-state step), in precise mode (the
   rows are built by the float64 library) and with MW_B200_SNAPSHOT_F32=1, next to one `step_torch` of the same envs.
2. The fresh-goal loop: DISABLED autoreset, every step followed by `reset_goals_torch` of the envs it ended, at goals
   drawn up front with `sample_goals`; env steps/s against `step_torch` under SAME_STEP autoreset on the same envs.
Times come from CUDA events around back-to-back calls after a warm-up.  Prints one JSON line with the card name, power
limit and max SM clock, and writes it to <out>/goal_reset_timing.json when an output directory is given.  Usage (on a GPU):
    python scripts/gpu_goal_reset_timing.py [out_dir]"""
import json, os, sys

import numpy as np
import torch

from gpu_timing_common import card, steady_env, timed

OUT = sys.argv[1] if len(sys.argv) > 1 else None
N = 4096


def steady(**kw):
    env = steady_env("MT50", N, use_one_hot=True, **kw)
    rng = np.random.default_rng(1)
    acts = [torch.from_numpy(rng.uniform(-1, 1, size=(N, 4)).astype(np.float32)).cuda() for _ in range(16)]
    for i in range(20):
        out = env.step_torch(acts[i % 16])
        if env.autoreset_mode == "Disabled":
            env.reset_torch(torch.logical_or(out[2], out[3]).bool())
    return env, acts


res = {"card": card(), "n_envs": N}
env, acts = steady()
k = [0]


def step():
    env.step_torch(acts[k[0] % 16]); k[0] += 1


res["step_torch_ms"] = step_ms = timed(step, 50)
rv, rv1 = (torch.from_numpy(x).cuda() for x in env.sample_goals(np.random.default_rng(2)))
everyone = torch.ones(N, dtype=torch.bool, device="cuda")
few = torch.zeros(N, dtype=torch.bool, device="cuda")
few[torch.from_numpy(np.random.default_rng(3).choice(N, 8, replace=False))] = True
for mode, f32 in (("precise", "0"), ("f32", "1")):
    os.environ["MW_B200_SNAPSHOT_F32"] = f32
    r = {"all_ms": timed(lambda: env.reset_goals_torch(rv, everyone, rv1), 3, warm=1),
         "8_envs_ms": timed(lambda: env.reset_goals_torch(rv, few, rv1), 10, warm=2)}
    r["all_over_step"], r["8_envs_over_step"] = r["all_ms"] / step_ms, r["8_envs_ms"] / step_ms
    res[mode] = r
os.environ.pop("MW_B200_SNAPSHOT_F32")
assert not env.engine.faults().any()
env.close()

# fresh-goal loop (DISABLED) against SAME_STEP step_torch on the same envs
env, acts = steady(autoreset_mode="Disabled")
pool = [env.sample_goals(np.random.default_rng(10 + i)) for i in range(4)]
P = torch.from_numpy(np.stack([p[0] for p in pool])).cuda()
P1 = torch.from_numpy(np.stack([p[1] for p in pool])).cuda()
count = torch.zeros(N, dtype=torch.long, device="cuda")
ar = torch.arange(N, device="cuda")
ends = torch.zeros((), dtype=torch.long, device="cuda")


def loop_step():
    out = env.step_torch(acts[k[0] % 16]); k[0] += 1
    ended = torch.logical_or(out[2], out[3]).bool()
    i = count % len(pool)
    env.reset_goals_torch(P[i, ar].contiguous(), ended, P1[i, ar].contiguous())
    count.add_(ended)
    ends.add_(ended.sum())


LOOP = 100
loop_ms = timed(loop_step, LOOP, warm=3)
n_ends = int(ends.item())
assert not env.engine.faults().any()
env.close()
res["fresh_goal_loop"] = {"steps": LOOP, "episode_ends_per_step": n_ends / (LOOP + 3), "ms_per_step": loop_ms,
                          "env_steps_per_s": N / (loop_ms * 1e-3), "same_step_env_steps_per_s": N / (step_ms * 1e-3)}
line = json.dumps(res)
print(line)
if OUT:
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "goal_reset_timing.json"), "w") as f:
        f.write(line + "\n")
