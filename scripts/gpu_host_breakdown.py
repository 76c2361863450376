"""Where the numpy-API step spends host time around the kernel (MT50 @ 4096, steady state)."""
import time, numpy as np, torch
from types import SimpleNamespace
from gpu_timing_common import card
from bench import build_env, stagger
print("card:", card())
env, names, _, _ = build_env(SimpleNamespace(benchmark="MT50", envs_per_gpu=4096, seed=42), 0, 0)
N = env.num_envs
env.reset(); stagger(env, 0)
rng = np.random.default_rng(1)
acts = [rng.uniform(-1, 1, size=(N, 4)).astype(np.float32) for _ in range(16)]
for i in range(500): env.step(acts[i % 16])          # same pre-roll as bench.py: steady-state contact load
marks = []
orig = torch.cuda.Stream.synchronize
def sync(self):
    t0 = time.perf_counter(); orig(self); marks.append((t0, time.perf_counter()))
torch.cuda.Stream.synchronize = sync
rows = []
ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(100)]
for i in range(100):
    ev[i][0].record()
    t0 = time.perf_counter(); env.step(acts[i % 16]); t1 = time.perf_counter()
    ev[i][1].record()
    s0, s1 = marks[-1]
    rows.append((s0 - t0, s1 - s0, t1 - s1, t1 - t0))
torch.cuda.synchronize()
r = np.array(rows) * 1e3
gpu = np.array([a.elapsed_time(b) for a, b in ev])
print(f"numpy step {r[:,3].mean():.3f} ms = before sync {r[:,0].mean():.3f} (launch + shadow work) + sync wait {r[:,1].mean():.3f} + after sync {r[:,2].mean():.3f}")
print(f"GPU busy per step (events around the call, includes copies) {gpu.mean():.3f} ms")
env.enable_device_sampler()
a = torch.from_numpy(acts[0]).to(env.device)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
for i in range(10): env.step_torch(a)
e0.record()
for i in range(100): env.step_torch(a)
e1.record(); torch.cuda.synchronize()
print(f"step_torch (device timed, hot L2): {e0.elapsed_time(e1) / 100:.3f} ms / step")
