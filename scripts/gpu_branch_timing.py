"""Device-timed saved states (k_save_states / k_load_states) and an MPPI-shaped planning loop.

1. MT50 x 4096 in steady state (episode phases staggered as in bench.py, 20 steps in): saving every env, loading every
   env, and a fork in which every env loads the state of a random env of its own model.  Each is timed as the engine call
   alone (caller-owned buffers: the two kernels) and as the vector env's call (`save_states` allocates its buffers,
   `load_states_torch` also restores the observation and wrapper rows), next to one `step_torch` of the same envs.
   The bytes a row moves are counted from the kernels' accesses, and bandwidth = bytes / kernel time.
2. MPPI-shaped loop on one task: 64 source states x 64 branches = 4096 envs.  Each iteration forks every branch from its
   source (`load_states_torch`) and rolls it out for 30 `step_torch` steps.
Times come from CUDA events around `reps` back-to-back calls after a warm-up.  Prints one JSON line with the card name and
its power limit, and writes it to <out>/branch_timing.json when an output directory is given.  Usage (on a GPU):
    python scripts/gpu_branch_timing.py [reps] [out_dir]"""
import json, os, sys

import numpy as np
import torch

from gpu_timing_common import card, steady_env, timed

REPS = max(200, int(sys.argv[1]) if len(sys.argv) > 1 else 200)
OUT = sys.argv[2] if len(sys.argv) > 2 else None
N = 4096
REC, HINTS, IDX = 512, 128 * 16, 4           # state record, separating-axis hints, one int32


def steady(name, use_one_hot):
    env = steady_env(name, N, use_one_hot=use_one_hot)
    rng = np.random.default_rng(1)
    acts = [torch.from_numpy(rng.uniform(-1, 1, size=(N, 4)).astype(np.float32)).cuda() for _ in range(16)]
    for i in range(20):
        env.step_torch(acts[i % 16])
    return env, acts


def entry(ms, read, written):
    return {"ms": ms, "bytes_read": read, "bytes_written": written, "GB_per_s": (read + written) / (ms * 1e-3) / 1e9}


res = {"card": card(), "n_envs": N, "reps": REPS}
env, acts = steady("MT50", True)
eng = env.engine
st = env.save_states()
rng = np.random.default_rng(2)
model = np.asarray(eng.env_model)
fork = np.array([rng.choice(np.nonzero(model == model[e])[0]) for e in range(N)])
d_fork = torch.from_numpy(fork.astype(np.int32)).cuda()
k = [0]


def step():
    env.step_torch(acts[k[0] % 16]); k[0] += 1


step_ms = timed(step, max(20, REPS // 5))
# per row: save reads the record, the hints and the model slot and writes them; load also reads src and both model slots
save_b = N * (REC + HINTS + IDX)
load_rd, load_wr = N * (REC + HINTS + 3 * IDX), N * (REC + HINTS)
res["mt50"] = {
    "step_torch_ms": step_ms,
    "engine_save_all": entry(timed(lambda: eng.save_states(st.records, st.model, st.hints), REPS), save_b, save_b),
    "engine_load_all": entry(timed(lambda: eng.load_states(st.records, st.model, st.hints), REPS), load_rd - N * IDX, load_wr),
    "engine_fork_same_model": entry(timed(lambda: eng.load_states(st.records, st.model, st.hints, src=d_fork), REPS), load_rd, load_wr),
    "env_save_states_ms": timed(env.save_states, REPS),
    "env_load_states_torch_ms": timed(lambda: env.load_states_torch(st), REPS),
    "env_fork_ms": timed(lambda: env.load_states_torch(st, src=d_fork), REPS),
}
res["mt50"]["fork_over_step"] = res["mt50"]["env_fork_ms"] / step_ms
assert not eng.faults().any()
env.close()

# MPPI-shaped: branch b of source s = env 64 s + b restarts every iteration from env 64 s's saved state
task, H, B = "pick-place-v3", 30, 64
env, acts = steady(task, False)
st = env.save_states()
src = (torch.arange(N, device="cuda") // B) * B
plans = torch.rand(H, N, 4, device="cuda") * 2 - 1


def iteration():
    env.load_states_torch(st, src=src)
    for h in range(H):
        env.step_torch(plans[h])


fork_ms = timed(lambda: env.load_states_torch(st, src=src), REPS)
step_ms = timed(lambda: env.step_torch(plans[0]), max(20, REPS // 5))
it_ms = timed(iteration, max(5, REPS // 20), warm=2)
res["mppi"] = {"task": task, "sources": N // B, "branches": B, "horizon": H, "iteration_ms": it_ms, "fork_ms": fork_ms,
               "step_torch_ms": step_ms, "fork_over_step": fork_ms / step_ms, "env_steps_per_s": N * H / (it_ms * 1e-3)}
assert not env.engine.faults().any()
env.close()
line = json.dumps(res)
print(line)
if OUT:
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "branch_timing.json"), "w") as f:
        f.write(line + "\n")
