"""Device-timed state queries.

`query_torch()` on all envs of MT50 x 4096 in steady state (episode phases staggered as in bench.py, 20 steps in): the
observation frame only (kinematics pass), with 16 named frames, and with `touching=True` (full forward pass), next to
one `step_torch` of the same envs.  Times come from CUDA events around `reps` back-to-back calls after a warm-up.
Prints one JSON line with the card name, its power limit and max SM clock, and writes it to <out>/query_timing.json
when an output directory is given.  Usage (on a GPU):
    python scripts/gpu_query_timing.py [reps] [out_dir]"""
import json, os, sys

import numpy as np
import torch

from gpu_timing_common import card, steady_env, timed

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 100
OUT = sys.argv[2] if len(sys.argv) > 2 else None
N = 4096
BODIES = ("hand", "rightpad", "leftpad", "rightclaw", "leftclaw", "obj")
SITES = ("rightEndEffector", "leftEndEffector", "goal", "hole", "handle")
GEOMS = ("objGeom", "leftpad_geom", "rightpad_geom", "handle", "mug")       # 16 frames in all


def main():
    env = steady_env("MT50", N, use_one_hot=True)
    A = torch.from_numpy(np.random.default_rng(1).uniform(-1, 1, size=(N, 4)).astype(np.float32)).to(env.device)
    for _ in range(20):
        env.step_torch(A)
    st0 = env.engine.get_state()
    res = {"card": card(), "n_envs": N, "reps": REPS,
           "query_frame_ms": timed(lambda: env.query_torch(), REPS),
           "query_16_frames_ms": timed(lambda: env.query_torch(bodies=BODIES, sites=SITES, geoms=GEOMS), REPS),
           "query_touching_ms": timed(lambda: env.query_torch(touching=True), REPS)}
    env.engine.set_state(st0)
    res["step_ms"] = timed(lambda: env.step_torch(A), REPS)
    assert not env.engine.faults().any()
    env.close()
    line = json.dumps(res)
    print(line)
    if OUT:
        os.makedirs(OUT, exist_ok=True)
        with open(os.path.join(OUT, "query_timing.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
