"""What the device-timing scripts share: the card a time was measured on, a CUDA-event timer, and MT50-style envs with
their episode phases staggered as in bench.py.  Importing this module touches no CUDA."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    """The device's name from torch, and nvidia-smi's name, power limit and max SM clock."""
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q[0] if q else None}


def timed(fn, reps, warm=5):
    """ms per call of `fn`: CUDA events around `reps` back-to-back calls after `warm` calls."""
    import torch
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


def steady_env(name, n=4096, **make_kw):
    """make_mt_envs(name, seed=42, num_envs=n, **make_kw), reset, with the episode phases of bench.stagger(env, 0)."""
    import bench
    from metaworld_b200.vector_env import make_mt_envs
    env = make_mt_envs(name, seed=42, num_envs=n, **make_kw)
    env.reset()
    bench.stagger(env, 0)
    return env
